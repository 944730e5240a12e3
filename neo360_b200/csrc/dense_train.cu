// Training form of the dense MLPs of vanilla NeRF (NeRFMLP, 8 x 256) and Mip-NeRF 360 (PropMLP 4 x 256, NeRFMLP 8 x 1024) on Hopper
// tensor cores: bf16 operands, fp32 accumulation, no floating-point atomics (neo360_b200.dense_train._MLPTrainTC drives it per layer).
// The three products run in gemm_tc.cu's one TMA / wgmma main loop (gemm_bf16, dgrad_bf16, wgrad_bf16_partials); this file holds
// their entry points and the small kernels around them:
//   pack_t          W^T in bf16 (the data gradient's B operand), from the fp32 master weights
//   relu_rank1      dz = bf16(g w^T) [X > 0]: the gradient into the last trunk activation of an MLP without a bottleneck (PropMLP)
//   colsum          per-split column sums of a bf16 row gradient (bias gradients)
//   wgrad_reduce    the fixed-order sum of the weight gradient's split partials and of the column sums
// The weight gradient splits the rows into a number of ranges that depends only on (M, N, K) (splits_of), so two calls on any device
// sum in the same order and are bit-identical.
#include "common.cuh"
#include <cuda_bf16.h>
#include <algorithm>

namespace neo {
namespace dtrain {

constexpr int kColSplits = 64;                                   // row ranges of the column sums
constexpr long long kMaxPartialBytes = 32ll << 20;               // bound on the weight gradient's split partials

__global__ void pack_t_kernel(const float* __restrict__ in, long long rows, long long ld_in, __nv_bfloat16* __restrict__ out, int cols_out,
                              long long ld_out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * cols_out) return;
    const long long r = idx % rows;
    const int c = (int)(idx / rows);
    out[c * ld_out + r] = __float2bfloat16_rn(in[r * ld_in + c]);
}

__global__ void relu_rank1_kernel(const float* __restrict__ g, const float* __restrict__ w, const __nv_bfloat16* __restrict__ X, long long ldx,
                                  long long M, int N, __nv_bfloat16* __restrict__ out, long long ldo) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= M * N) return;
    const long long r = idx / N;
    const int c = (int)(idx % N);
    const float v = __bfloat162float(X[r * ldx + c]) > 0.f ? g[r] * w[c] : 0.f;
    out[r * ldo + c] = __float2bfloat16_rn(v);
}

// part[s][c], part[s][c + 1] = sums of Y[r][c], Y[r][c + 1] over the rows of split s, in row order
__global__ void colsum_kernel(const __nv_bfloat16* __restrict__ Y, long long ld, long long M, int N, float* __restrict__ part) {
    const int c = 2 * (blockIdx.x * blockDim.x + threadIdx.x);
    if (c >= N) return;
    const int s = blockIdx.y;
    const long long r0 = M * s / kColSplits, r1 = M * (s + 1) / kColSplits;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll 4
    for (long long r = r0; r < r1; ++r) {
        const float2 y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(Y + r * ld + c));
        a0 += y.x;
        a1 += y.y;
    }
    part[(long long)s * N + c] = a0;
    part[(long long)s * N + c + 1] = a1;
}

__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int splits, int N, int K, int k_valid, float* __restrict__ dW,
                                    const float* __restrict__ cpart, float* __restrict__ db) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long nw = (long long)N * k_valid;
    if (idx < nw) {
        const int n = (int)(idx / k_valid), k = (int)(idx % k_valid);
        float s = 0.f;
        for (int z = 0; z < splits; ++z) s += part[(long long)z * N * K + (long long)n * K + k];
        dW[idx] = s;
    } else if (db && idx < nw + N) {
        const int n = (int)(idx - nw);
        float s = 0.f;
        for (int z = 0; z < kColSplits; ++z) s += cpart[(long long)z * N + n];
        db[n] = s;
    }
}

// enough 128 x BN tiles for two per SM slot on a large GPU, as many as the rows allow, within kMaxPartialBytes: a function of the shape only
static int splits_of(long long M, int N, int K) {
    const long long tiles = (long long)((N + 127) / 128) * (K % 128 == 0 ? K / 128 : K / 64);
    const long long kblocks = (M + 63) / 64;
    long long s = (256 + tiles - 1) / tiles;
    s = std::min(s, kblocks);
    s = std::min(s, kMaxPartialBytes / ((long long)N * K * 4));
    return (int)std::max(s, 1ll);
}
static size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }
static size_t wgrad_ws(long long M, int N, int K) {
    return align_up((size_t)splits_of(M, N, K) * N * K * 4) + (size_t)kColSplits * N * 4;
}
static bool wgrad_shape_ok(long long M, int N, int K) {
    return M > 0 && N > 0 && K > 0 && N % 64 == 0 && K % 64 == 0 && (long long)N * K * 4 <= kMaxPartialBytes;
}

}  // namespace dtrain
}  // namespace neo

using namespace neo::dtrain;

extern "C" int neo_tc_gemm_bf16(const void* A, long long lda, const void* W, long long ldw, const float* bias, void* C, long long ldc,
                                long long M, int N, int K, int epilogue, void* stream) {
    return neo::gemm_bf16(A, lda, W, ldw, bias, C, ldc, M, N, K, epilogue, (cudaStream_t)stream);
}

extern "C" int neo_tc_dgrad_bf16(const void* dY, long long ldy, const void* Wt, long long ldwt, const void* X, long long ldx,
                                 const float* g_sig, const float* w_sig, void* dX, long long lddx, long long M, int N, int K, void* stream) {
    return neo::dgrad_bf16(dY, ldy, Wt, ldwt, X, ldx, g_sig, w_sig, dX, lddx, M, N, K, (cudaStream_t)stream);
}

extern "C" size_t neo_tc_wgrad_bf16_workspace_bytes(long long M, int N, int K) {
    if (!wgrad_shape_ok(M, N, K)) {
        neo::set_error("wgrad_bf16: need M, N, K > 0, N %% 64 == 0, K %% 64 == 0 and N*K*4 <= %lld (got M=%lld N=%d K=%d)", kMaxPartialBytes, M, N, K);
        return 0;
    }
    return wgrad_ws(M, N, K);
}

extern "C" int neo_tc_wgrad_bf16(const void* dY, long long ldy, const void* X, long long ldx, long long M, int N, int K, float* dW, int k_valid,
                                 float* db, void* ws, size_t ws_bytes, void* stream) {
    if (!wgrad_shape_ok(M, N, K) || ldy < N || ldx < K || (ldy % 8) || (ldx % 8) || k_valid < 1 || k_valid > K) {
        neo::set_error("wgrad_bf16: need M, N, K > 0, N %% 64 == 0, K %% 64 == 0, N*K*4 <= %lld, row strides %% 8 == 0, ldy >= N, ldx >= K "
                       "and 0 < k_valid <= K (got M=%lld N=%d K=%d ldy=%lld ldx=%lld k_valid=%d)", kMaxPartialBytes, M, N, K, ldy, ldx, k_valid);
        return NEO_ERR_INVALID;
    }
    if (!dY || !X || !dW || !ws) { neo::set_error("wgrad_bf16: NULL buffer"); return NEO_ERR_INVALID; }
    if ((reinterpret_cast<uintptr_t>(dY) | reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(ws)) & 15) {
        neo::set_error("wgrad_bf16: dY, X and the workspace must be 16-byte aligned"); return NEO_ERR_INVALID;
    }
    if (ws_bytes < wgrad_ws(M, N, K)) { neo::set_error("wgrad_bf16: workspace of %zu bytes, %zu needed", ws_bytes, wgrad_ws(M, N, K)); return NEO_ERR_WORKSPACE; }
    cudaStream_t s = (cudaStream_t)stream;
    const int splits = splits_of(M, N, K);
    float* part = (float*)ws;
    float* cpart = (float*)((unsigned char*)ws + align_up((size_t)splits * N * K * 4));
    int rc = neo::wgrad_bf16_partials(dY, ldy, X, ldx, M, N, K, splits, part, s);
    if (rc) return rc;
    if (db) {
        colsum_kernel<<<dim3((unsigned)((N / 2 + 127) / 128), kColSplits), 128, 0, s>>>((const __nv_bfloat16*)dY, ldy, M, N, cpart);
        NEO_LAUNCH_CHECK("colsum_kernel");
    }
    const long long total = (long long)N * k_valid + (db ? N : 0);
    wgrad_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(part, splits, N, K, k_valid, dW, cpart, db);
    NEO_LAUNCH_CHECK("wgrad_reduce_kernel");
    return NEO_OK;
}

extern "C" int neo_tc_pack_bf16(const float* in, long long rows, int cols_in, long long ld_in, void* out, int cols_out, long long ld_out,
                                int transpose, void* stream) {
    const bool ok = rows > 0 && cols_in > 0 && cols_out > 0 && ld_in >= cols_in && (transpose == 0 || transpose == 1) &&
                    (transpose ? cols_out <= cols_in && ld_out >= rows : ld_out >= cols_out);
    if (!ok) {
        neo::set_error("pack_bf16: need rows, cols > 0, ld_in >= cols_in, transpose 0 or 1, and ld_out >= cols_out (transpose 0) or "
                       "cols_out <= cols_in and ld_out >= rows (transpose 1) (got rows=%lld cols_in=%d ld_in=%lld cols_out=%d ld_out=%lld "
                       "transpose=%d)", rows, cols_in, ld_in, cols_out, ld_out, transpose);
        return NEO_ERR_INVALID;
    }
    if (!in || !out) { neo::set_error("pack_bf16: NULL buffer"); return NEO_ERR_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    if (!transpose) return neo::f32_to_f16_pad(in, rows, cols_in, ld_in, out, cols_out, ld_out, s, 1);
    const long long total = rows * cols_out;
    pack_t_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, rows, ld_in, (__nv_bfloat16*)out, cols_out, ld_out);
    NEO_LAUNCH_CHECK("pack_t_kernel");
    return NEO_OK;
}

extern "C" int neo_tc_relu_rank1_bf16(const float* g, const float* w, const void* X, long long ldx, long long M, int N, void* out, long long ldo,
                                      void* stream) {
    if (M <= 0 || N <= 0 || ldx < N || ldo < N) {
        neo::set_error("relu_rank1_bf16: need M, N > 0, ldx >= N and ldo >= N (got M=%lld N=%d ldx=%lld ldo=%lld)", M, N, ldx, ldo);
        return NEO_ERR_INVALID;
    }
    if (!g || !w || !X || !out) { neo::set_error("relu_rank1_bf16: NULL buffer"); return NEO_ERR_INVALID; }
    const long long total = M * N;
    relu_rank1_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g, w, (const __nv_bfloat16*)X, ldx, M, N,
                                                                                        (__nv_bfloat16*)out, ldo);
    NEO_LAUNCH_CHECK("relu_rank1_kernel");
    return NEO_OK;
}

extern "C" int neo_tc_rowdot_bf16(const void* H, long long ld, int K, const float* W, const float* b, int N, long long M, float* out, void* stream) {
    return neo::launch_rowdot_f16(H, ld, K, W, b, N, M, out, (cudaStream_t)stream, 1);
}
