// Geometry export: the lattice rays that evaluate a NeO-360 foreground field on a density grid, marching tetrahedra over that grid,
// and the grid's normals at the mesh vertices.  Contracts are in include/neo360_b200.h; DESIGN.md section 10 gives the reasoning.
//
// Marching tetrahedra on the Kuhn subdivision: every cell is cut into the 6 tetrahedra {0, e_a, e_a + e_b, 1} (a, b, c a permutation of
// the axes), which all share the cell's main diagonal and cut each face along the diagonal through its lowest corner.  Neighbouring
// cells therefore agree on every face, and a tetrahedron has no ambiguous case, so the level set of a grid whose inside region does not
// touch the grid boundary is a closed, consistently oriented surface.
//
// Every edge of the subdivision joins a lattice point p to p + e, e a non-zero 0/1 vector.  Point p owns its 7 such edges, in the type
// order +x, +y, +z, +x+y, +x+z, +y+z, +x+y+z; vertex ids follow (point, type) order.  Counting and writing are two passes over the
// points, one thread per point, with an exclusive scan of per-block totals in between (two levels of 1024: at most 2^20 blocks); a
// block's threads take their offsets from a block scan.  Integer sums are exact in any order and nothing else is reduced, so the output
// is a function of the inputs alone.
#include "common.cuh"
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

namespace neo {
namespace {

constexpr int kBlock = 256;
constexpr long long kMaxPoints = 1LL << 28;     // 12 triangles per cell keep every count and offset below 2^32
constexpr int kScan = 1024;                     // kMaxPoints / kBlock = kScan * kScan block totals

struct GridDev {
    int nx, ny, nz;
    float o[3], h[3];
};

// corner code = dx | dy << 1 | dz << 2 of the corner offset inside a cell
__constant__ int kEdgeCode[7] = {1, 2, 4, 3, 5, 6, 7};               // owned edge type -> offset code
__constant__ int kTypeOfCode[8] = {-1, 0, 1, 3, 2, 4, 5, 6};         // offset code -> owned edge type
// the 6 Kuhn tetrahedra, each listed in positive orientation (det(c1 - c0, c2 - c0, c3 - c0) > 0)
__constant__ int kTet[6][4] = {{0, 1, 3, 7}, {1, 0, 5, 7}, {2, 0, 3, 7}, {0, 2, 6, 7}, {0, 4, 5, 7}, {4, 0, 6, 7}};

__device__ __forceinline__ float lattice(const GridDev& g, int axis, int idx) { return add_(g.o[axis], mul_((float)idx, g.h[axis])); }

__device__ __forceinline__ void decode(const GridDev& g, long long p, int& i, int& j, int& k) {
    i = (int)(p % g.nx);
    const long long q = p / g.nx;
    j = (int)(q % g.ny);
    k = (int)(q / g.ny);
}

__device__ __forceinline__ long long code_offset(const GridDev& g, int c) {
    return (long long)((c >> 2) & 1) * g.ny * g.nx + (long long)((c >> 1) & 1) * g.nx + (c & 1);
}

// bit t set: owned edge t of point p exists and its endpoints lie on different sides (inside = sigma >= iso)
__device__ unsigned edge_mask(const float* __restrict__ sig, const GridDev& g, long long p, int i, int j, int k, float iso) {
    const bool a = sig[p] >= iso;
    unsigned m = 0;
#pragma unroll
    for (int t = 0; t < 7; ++t) {
        const int c = kEdgeCode[t];
        if (i + (c & 1) >= g.nx || j + ((c >> 1) & 1) >= g.ny || k + ((c >> 2) & 1) >= g.nz) continue;
        if ((sig[p + code_offset(g, c)] >= iso) != a) m |= 1u << t;
    }
    return m;
}

// inside bits of the 8 corners of the cell whose lowest corner is p; 0 and triangle count 0 when p starts no cell
__device__ unsigned cell_bits(const float* __restrict__ sig, const GridDev& g, long long p, int i, int j, int k, float iso, int& tris) {
    tris = 0;
    if (i + 1 >= g.nx || j + 1 >= g.ny || k + 1 >= g.nz) return 0;
    unsigned bits = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) bits |= (unsigned)(sig[p + code_offset(g, c)] >= iso) << c;
#pragma unroll
    for (int t = 0; t < 6; ++t) {
        const int n = ((bits >> kTet[t][0]) & 1) + ((bits >> kTet[t][1]) & 1) + ((bits >> kTet[t][2]) & 1) + ((bits >> kTet[t][3]) & 1);
        tris += (n == 2) ? 2 : (n == 1 || n == 3) ? 1 : 0;
    }
    return bits;
}

__device__ __forceinline__ bool odd_perm(const int* q) {
    int inv = 0;
    for (int a = 0; a < 4; ++a)
        for (int b = a + 1; b < 4; ++b) inv += q[a] > q[b];
    return inv & 1;
}

// Triangles of tetrahedron t with local inside mask m, as pairs of local corners per triangle vertex; returns their number (0..2).
// One inside corner a: with (a, j, k, l) an even permutation (j < k < l, k and l swapped if needed), the triangle (aj, ak, al).  One
// outside corner a: (aj, al, ak).  Inside i0 < i1, outside o0, o1 with (i0, i1, o0, o1) even: (i0o0, i0o1, i1o1), (i0o0, i1o1, i1o0).
// Each faces the outside corners, i.e. winds counter-clockwise seen from lower sigma.
__device__ int tet_tris(unsigned m, int (&e)[2][3][2]) {
    const int n = __popc(m);
    if (n == 0 || n == 4) return 0;
    if (n == 2) {
        int q[4], ni = 0, no = 2;
        for (int c = 0; c < 4; ++c) q[((m >> c) & 1) ? ni++ : no++] = c;
        if (odd_perm(q)) { const int s = q[2]; q[2] = q[3]; q[3] = s; }
        const int i0 = q[0], i1 = q[1], o0 = q[2], o1 = q[3];
        const int tri[2][3][2] = {{{i0, o0}, {i0, o1}, {i1, o1}}, {{i0, o0}, {i1, o1}, {i1, o0}}};
        for (int a = 0; a < 2; ++a)
            for (int b = 0; b < 3; ++b) { e[a][b][0] = tri[a][b][0]; e[a][b][1] = tri[a][b][1]; }
        return 2;
    }
    const unsigned lone_bit = (n == 1) ? m : (~m & 15u);
    int q[4], r = 1;
    q[0] = __ffs(lone_bit) - 1;
    for (int c = 0; c < 4; ++c)
        if (c != q[0]) q[r++] = c;
    if (odd_perm(q)) { const int s = q[2]; q[2] = q[3]; q[3] = s; }
    const int a = q[0];
    e[0][0][0] = a; e[0][0][1] = q[1];
    e[0][1][0] = a; e[0][1][1] = (n == 1) ? q[2] : q[3];
    e[0][2][0] = a; e[0][2][1] = (n == 1) ? q[3] : q[2];
    return 1;
}

__global__ void __launch_bounds__(kBlock) mt_count_kernel(const float* __restrict__ sig, GridDev g, float iso, long long P,
                                                          unsigned* __restrict__ blk_v, unsigned* __restrict__ blk_t) {
    using Reduce = cub::BlockReduce<unsigned, kBlock>;
    __shared__ typename Reduce::TempStorage rv, rt;
    const long long p = (long long)blockIdx.x * kBlock + threadIdx.x;
    unsigned nv = 0;
    int nt = 0;
    if (p < P) {
        int i, j, k;
        decode(g, p, i, j, k);
        nv = __popc(edge_mask(sig, g, p, i, j, k, iso));
        cell_bits(sig, g, p, i, j, k, iso, nt);
    }
    const unsigned sv = Reduce(rv).Sum(nv);
    const unsigned st = Reduce(rt).Sum((unsigned)nt);
    if (threadIdx.x == 0) { blk_v[blockIdx.x] = sv; blk_t[blockIdx.x] = st; }
}

// exclusive scan of the block totals inside each run of kScan blocks, and the run's sum
__global__ void __launch_bounds__(kScan) scan_runs_kernel(const unsigned* __restrict__ blk_v, const unsigned* __restrict__ blk_t, long long nb,
                                                          unsigned* __restrict__ off_v, unsigned* __restrict__ off_t, unsigned* __restrict__ run_v,
                                                          unsigned* __restrict__ run_t) {
    using Scan = cub::BlockScan<unsigned, kScan>;
    __shared__ typename Scan::TempStorage tv, tt;
    const long long b = (long long)blockIdx.x * kScan + threadIdx.x;
    unsigned ov, ot, sv, st;
    Scan(tv).ExclusiveSum(b < nb ? blk_v[b] : 0u, ov, sv);
    Scan(tt).ExclusiveSum(b < nb ? blk_t[b] : 0u, ot, st);
    if (b < nb) { off_v[b] = ov; off_t[b] = ot; }
    if (threadIdx.x == 0) { run_v[blockIdx.x] = sv; run_t[blockIdx.x] = st; }
}
// in place: exclusive scan of the (at most kScan) run sums; totals = V and F
__global__ void __launch_bounds__(kScan) scan_run_sums_kernel(unsigned* __restrict__ run_v, unsigned* __restrict__ run_t, int n_runs,
                                                              unsigned* __restrict__ totals) {
    using Scan = cub::BlockScan<unsigned, kScan>;
    __shared__ typename Scan::TempStorage tv, tt;
    const int r = threadIdx.x;
    unsigned ov, ot, sv, st;
    Scan(tv).ExclusiveSum(r < n_runs ? run_v[r] : 0u, ov, sv);
    Scan(tt).ExclusiveSum(r < n_runs ? run_t[r] : 0u, ot, st);
    if (r < n_runs) { run_v[r] = ov; run_t[r] = ot; }
    if (r == 0) { totals[0] = sv; totals[1] = st; }
}

__global__ void __launch_bounds__(kBlock) mt_vertex_kernel(const float* __restrict__ sig, GridDev g, float iso, long long P,
                                                           const unsigned* __restrict__ off_v, const unsigned* __restrict__ run_v,
                                                           unsigned* __restrict__ vbase,
                                                           unsigned char* __restrict__ vmask, float* __restrict__ verts, long long n_verts) {
    using Scan = cub::BlockScan<unsigned, kBlock>;
    __shared__ typename Scan::TempStorage ts;
    const long long p = (long long)blockIdx.x * kBlock + threadIdx.x;
    int i = 0, j = 0, k = 0;
    unsigned m = 0;
    if (p < P) {
        decode(g, p, i, j, k);
        m = edge_mask(sig, g, p, i, j, k, iso);
    }
    unsigned local;
    Scan(ts).ExclusiveSum((unsigned)__popc(m), local);
    if (p >= P) return;
    const unsigned base = run_v[blockIdx.x / kScan] + off_v[blockIdx.x] + local;
    vbase[p] = base;
    vmask[p] = (unsigned char)m;
    if (!m) return;
    const float sa = sig[p];
    const float pa[3] = {lattice(g, 0, i), lattice(g, 1, j), lattice(g, 2, k)};
    unsigned id = base;
    for (int t = 0; t < 7; ++t) {
        if (!((m >> t) & 1)) continue;
        const int c = kEdgeCode[t];
        const float sb = sig[p + code_offset(g, c)];
        const float pb[3] = {lattice(g, 0, i + (c & 1)), lattice(g, 1, j + ((c >> 1) & 1)), lattice(g, 2, k + ((c >> 2) & 1))};
        // the stated operation order: w = (iso - sa) / (sb - sa), x = pa + w * (pb - pa), each step rounded to nearest
        const float w = __fdiv_rn(sub_(iso, sa), sub_(sb, sa));
        if ((long long)id < n_verts)
            for (int a = 0; a < 3; ++a) verts[3 * (long long)id + a] = add_(pa[a], mul_(w, sub_(pb[a], pa[a])));
        ++id;
    }
}

__global__ void __launch_bounds__(kBlock) mt_face_kernel(const float* __restrict__ sig, GridDev g, float iso, long long P,
                                                         const unsigned* __restrict__ off_t, const unsigned* __restrict__ run_t,
                                                         const unsigned* __restrict__ vbase,
                                                         const unsigned char* __restrict__ vmask, int* __restrict__ faces, long long n_faces) {
    using Scan = cub::BlockScan<unsigned, kBlock>;
    __shared__ typename Scan::TempStorage ts;
    const long long p = (long long)blockIdx.x * kBlock + threadIdx.x;
    int nt = 0;
    unsigned bits = 0;
    if (p < P) {
        int i, j, k;
        decode(g, p, i, j, k);
        bits = cell_bits(sig, g, p, i, j, k, iso, nt);
    }
    unsigned local;
    Scan(ts).ExclusiveSum((unsigned)nt, local);
    if (p >= P || !nt) return;
    unsigned f = run_t[blockIdx.x / kScan] + off_t[blockIdx.x] + local;
    for (int t = 0; t < 6; ++t) {
        unsigned m = 0;
        for (int c = 0; c < 4; ++c) m |= ((bits >> kTet[t][c]) & 1u) << c;
        int e[2][3][2];
        const int n = tet_tris(m, e);
        for (int a = 0; a < n; ++a, ++f) {
            if ((long long)f >= n_faces) continue;
            for (int b = 0; b < 3; ++b) {
                const int c0 = kTet[t][e[a][b][0]], c1 = kTet[t][e[a][b][1]];
                const int lo = ((c0 & c1) == c0) ? c0 : c1;       // the corners of a Kuhn tetrahedron form a chain: one is a subset
                const long long q = p + code_offset(g, lo);
                const int type = kTypeOfCode[c0 ^ c1];
                faces[3 * (long long)f + b] = (int)(vbase[q] + __popc(vmask[q] & ((1u << type) - 1u)));
            }
        }
    }
}

// Central differences of sigma at lattice point (i, j, k), one-sided on the grid's faces; d = sigma difference over the coordinate span.
__device__ void lattice_grad(const float* __restrict__ sig, const GridDev& g, int i, int j, int k, float* gr) {
    const int idx[3] = {i, j, k}, n[3] = {g.nx, g.ny, g.nz};
    const long long stride[3] = {1, g.nx, (long long)g.nx * g.ny};
    const long long p = k * stride[2] + j * stride[1] + i;
    for (int a = 0; a < 3; ++a) {
        const int lo = idx[a] > 0 ? idx[a] - 1 : 0, hi = idx[a] < n[a] - 1 ? idx[a] + 1 : n[a] - 1;
        gr[a] = (sig[p + (hi - idx[a]) * stride[a]] - sig[p + (lo - idx[a]) * stride[a]]) / ((float)(hi - lo) * g.h[a]);
    }
}

__global__ void grid_normals_kernel(const float* __restrict__ sig, GridDev g, const float* __restrict__ verts, long long n,
                                    float* __restrict__ normals) {
    const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    const int n_ax[3] = {g.nx, g.ny, g.nz};
    int c0[3];
    float f[3];
    for (int a = 0; a < 3; ++a) {
        const float u = (verts[3 * v + a] - g.o[a]) / g.h[a];
        int ci = (int)floorf(u);
        ci = ci < 0 ? 0 : (ci > n_ax[a] - 2 ? n_ax[a] - 2 : ci);
        c0[a] = ci;
        f[a] = fminf(fmaxf(u - (float)ci, 0.f), 1.f);
    }
    float gs[3] = {0.f, 0.f, 0.f};
    for (int c = 0; c < 8; ++c) {
        const int dx = c & 1, dy = (c >> 1) & 1, dz = (c >> 2) & 1;
        const float w = (dx ? f[0] : 1.f - f[0]) * (dy ? f[1] : 1.f - f[1]) * (dz ? f[2] : 1.f - f[2]);
        float gr[3];
        lattice_grad(sig, g, c0[0] + dx, c0[1] + dy, c0[2] + dz, gr);
        for (int a = 0; a < 3; ++a) gs[a] += w * gr[a];
    }
    const float len = sqrtf(gs[0] * gs[0] + gs[1] * gs[1] + gs[2] * gs[2]);
    const float inv = len > 0.f ? -1.f / len : 0.f;
    for (int a = 0; a < 3; ++a) normals[3 * v + a] = gs[a] * inv;
}

__global__ void grid_rays_kernel(GridDev g, long long row0, int n_rows, float* __restrict__ o, float* __restrict__ d, float* __restrict__ t) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)n_rows * g.nx) return;
    const int r = (int)(e / g.nx), i = (int)(e % g.nx);
    t[e] = mul_((float)i, g.h[0]);
    if (i) return;
    const long long row = row0 + r;
    o[3 * r + 0] = g.o[0];
    o[3 * r + 1] = lattice(g, 1, (int)(row % g.ny));
    o[3 * r + 2] = lattice(g, 2, (int)(row / g.ny));
    d[3 * r + 0] = 1.f; d[3 * r + 1] = 0.f; d[3 * r + 2] = 0.f;
}

__global__ void grid_mask_sphere_kernel(GridDev g, long long row0, int n_rows, float* __restrict__ sig) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)n_rows * g.nx) return;
    const long long row = row0 + e / g.nx;
    const float x = lattice(g, 0, (int)(e % g.nx)), y = lattice(g, 1, (int)(row % g.ny)), z = lattice(g, 2, (int)(row / g.ny));
    if (add_(add_(mul_(x, x), mul_(y, y)), mul_(z, z)) > 1.0f) sig[e] = 0.f;
}

int check_grid(const char* who, const NeoGrid* grid, GridDev& g, long long& P) {
    if (!grid) { set_error("%s: NULL grid", who); return NEO_ERR_INVALID; }
    if (grid->nx < 2 || grid->ny < 2 || grid->nz < 2) {
        set_error("%s: the grid needs at least 2 points per axis (got %d x %d x %d)", who, grid->nx, grid->ny, grid->nz);
        return NEO_ERR_INVALID;
    }
    P = (long long)grid->nx * grid->ny * grid->nz;
    if (P > kMaxPoints) { set_error("%s: %lld grid points exceed 2^28", who, P); return NEO_ERR_INVALID; }
    g.nx = grid->nx; g.ny = grid->ny; g.nz = grid->nz;
    for (int a = 0; a < 3; ++a) {
        if (!isfinite(grid->origin[a]) || !isfinite(grid->step[a]) || !(grid->step[a] > 0.f)) {
            set_error("%s: origin must be finite and step finite and positive (axis %d: %g, %g)", who, a, grid->origin[a], grid->step[a]);
            return NEO_ERR_INVALID;
        }
        g.o[a] = grid->origin[a];
        g.h[a] = grid->step[a];
    }
    return NEO_OK;
}

// workspace blocks: per-block totals and offsets, per-run offsets, V and F, then each point's first vertex id and edge mask
struct MTBuffers {
    unsigned *blk_v, *blk_t, *off_v, *off_t, *run_v, *run_t, *totals, *vbase;
    unsigned char* vmask;
    size_t total;
};

void mt_carve(void* ws, long long P, MTBuffers& b) {
    const long long nb = (P + kBlock - 1) / kBlock;
    Carve c{static_cast<unsigned char*>(ws), 0};
    b.blk_v = c.take<unsigned>(nb);
    b.blk_t = c.take<unsigned>(nb);
    b.off_v = c.take<unsigned>(nb);
    b.off_t = c.take<unsigned>(nb);
    b.run_v = c.take<unsigned>(kScan);
    b.run_t = c.take<unsigned>(kScan);
    b.totals = c.take<unsigned>(2);
    b.vbase = c.take<unsigned>(P);
    b.vmask = c.take<unsigned char>(P);
    b.total = c.used;
}

int mt_prepare(const char* who, const float* sigma, const NeoGrid* grid, float iso, void* ws, size_t ws_bytes, GridDev& g, long long& P,
               MTBuffers& b) {
    int rc = check_grid(who, grid, g, P);
    if (rc) return rc;
    if (!sigma || !ws) { set_error("%s: NULL sigma or workspace", who); return NEO_ERR_INVALID; }
    if (!isfinite(iso)) { set_error("%s: iso must be finite", who); return NEO_ERR_INVALID; }
    if ((reinterpret_cast<uintptr_t>(ws) & 255) != 0) { set_error("%s: the workspace must be 256-byte aligned", who); return NEO_ERR_INVALID; }
    mt_carve(ws, P, b);
    if (ws_bytes < b.total) { set_error("%s: workspace of %zu bytes, %zu needed", who, ws_bytes, b.total); return NEO_ERR_WORKSPACE; }
    return NEO_OK;
}

}  // namespace
}  // namespace neo

using namespace neo;

extern "C" size_t neo_mt_workspace_bytes(const NeoGrid* grid) {
    GridDev g;
    long long P;
    MTBuffers b;
    if (check_grid("neo_mt_workspace_bytes", grid, g, P)) return 0;
    mt_carve(nullptr, P, b);
    return b.total;
}

extern "C" int neo_mt_count(const float* sigma, const NeoGrid* grid, float iso, void* workspace, size_t workspace_bytes, int* n_verts,
                            int* n_faces, void* stream) {
    GridDev g;
    long long P;
    MTBuffers b;
    if (!n_verts || !n_faces) { set_error("neo_mt_count: NULL n_verts or n_faces"); return NEO_ERR_INVALID; }
    int rc = mt_prepare("neo_mt_count", sigma, grid, iso, workspace, workspace_bytes, g, P, b);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const long long nb = (P + kBlock - 1) / kBlock;
    mt_count_kernel<<<(unsigned)nb, kBlock, 0, s>>>(sigma, g, iso, P, b.blk_v, b.blk_t);
    NEO_LAUNCH_CHECK("mt_count_kernel");
    const int n_runs = (int)((nb + kScan - 1) / kScan);
    scan_runs_kernel<<<n_runs, kScan, 0, s>>>(b.blk_v, b.blk_t, nb, b.off_v, b.off_t, b.run_v, b.run_t);
    NEO_LAUNCH_CHECK("scan_runs_kernel");
    scan_run_sums_kernel<<<1, kScan, 0, s>>>(b.run_v, b.run_t, n_runs, b.totals);
    NEO_LAUNCH_CHECK("scan_run_sums_kernel");
    unsigned tot[2] = {0, 0};
    NEO_CUDA(cudaMemcpyAsync(tot, b.totals, sizeof(tot), cudaMemcpyDeviceToHost, s));
    NEO_CUDA(cudaStreamSynchronize(s));
    if (tot[0] > 0x7fffffffu || tot[1] > 0x7fffffffu) {
        set_error("neo_mt_count: %u vertices / %u faces exceed int32 indices", tot[0], tot[1]);
        return NEO_ERR_UNSUPPORTED;
    }
    *n_verts = (int)tot[0];
    *n_faces = (int)tot[1];
    return NEO_OK;
}

extern "C" int neo_mt_emit(const float* sigma, const NeoGrid* grid, float iso, void* workspace, size_t workspace_bytes, float* verts, int n_verts,
                           int* faces, int n_faces, void* stream) {
    GridDev g;
    long long P;
    MTBuffers b;
    int rc = mt_prepare("neo_mt_emit", sigma, grid, iso, workspace, workspace_bytes, g, P, b);
    if (rc) return rc;
    if (n_verts < 0 || n_faces < 0 || (n_verts > 0 && !verts) || (n_faces > 0 && !faces)) {
        set_error("neo_mt_emit: negative sizes, or NULL verts / faces with a non-zero size");
        return NEO_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const long long nb = (P + kBlock - 1) / kBlock;
    mt_vertex_kernel<<<(unsigned)nb, kBlock, 0, s>>>(sigma, g, iso, P, b.off_v, b.run_v, b.vbase, b.vmask, verts, n_verts);
    NEO_LAUNCH_CHECK("mt_vertex_kernel");
    mt_face_kernel<<<(unsigned)nb, kBlock, 0, s>>>(sigma, g, iso, P, b.off_t, b.run_t, b.vbase, b.vmask, faces, n_faces);
    NEO_LAUNCH_CHECK("mt_face_kernel");
    return NEO_OK;
}

extern "C" int neo_grid_normals(const float* sigma, const NeoGrid* grid, const float* verts, int n_verts, float* normals, void* stream) {
    GridDev g;
    long long P;
    int rc = check_grid("neo_grid_normals", grid, g, P);
    if (rc) return rc;
    if (n_verts < 0 || (n_verts > 0 && (!sigma || !verts || !normals))) {
        set_error("neo_grid_normals: negative n_verts, or NULL sigma / verts / normals");
        return NEO_ERR_INVALID;
    }
    if (n_verts == 0) return NEO_OK;
    grid_normals_kernel<<<(unsigned)((n_verts + 255) / 256), 256, 0, (cudaStream_t)stream>>>(sigma, g, verts, n_verts, normals);
    NEO_LAUNCH_CHECK("grid_normals_kernel");
    return NEO_OK;
}

extern "C" int neo_grid_rays(const NeoGrid* grid, long long row0, int n_rows, float* rays_o, float* dirs, float* t_vals, void* stream) {
    GridDev g;
    long long P;
    int rc = check_grid("neo_grid_rays", grid, g, P);
    if (rc) return rc;
    if (row0 < 0 || n_rows < 1 || row0 + n_rows > (long long)g.ny * g.nz || !rays_o || !dirs || !t_vals) {
        set_error("neo_grid_rays: rows [%lld, %lld) outside the grid's %lld, or a NULL output", row0, row0 + n_rows, (long long)g.ny * g.nz);
        return NEO_ERR_INVALID;
    }
    const long long n = (long long)n_rows * g.nx;
    grid_rays_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g, row0, n_rows, rays_o, dirs, t_vals);
    NEO_LAUNCH_CHECK("grid_rays_kernel");
    return NEO_OK;
}

extern "C" int neo_grid_mask_sphere(const NeoGrid* grid, long long row0, int n_rows, float* sigma_rows, void* stream) {
    GridDev g;
    long long P;
    int rc = check_grid("neo_grid_mask_sphere", grid, g, P);
    if (rc) return rc;
    if (row0 < 0 || n_rows < 1 || row0 + n_rows > (long long)g.ny * g.nz || !sigma_rows) {
        set_error("neo_grid_mask_sphere: rows [%lld, %lld) outside the grid's %lld, or NULL sigma", row0, row0 + n_rows, (long long)g.ny * g.nz);
        return NEO_ERR_INVALID;
    }
    const long long n = (long long)n_rows * g.nx;
    grid_mask_sphere_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g, row0, n_rows, sigma_rows);
    NEO_LAUNCH_CHECK("grid_mask_sphere_kernel");
    return NEO_OK;
}
