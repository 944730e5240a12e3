// Generic dense layer on Hopper tensor cores (sm_90a):  C[M][N] = act(A[M][K] . W[N][K]^T + bias)   fp16 operands, fp32 accumulate.
// A and W are K-major (row-major activations, nn.Linear weights), so both operands are staged by 2-D TMA tile loads
// (cp.async.bulk.tensor.2d, 128-byte swizzle) straight into the layout wgmma reads.  Used by the tensor-core paths of the wide
// MLPs: Mip-NeRF 360's 8 x 1024 NeRF MLP and 4 x 256 proposal MLPs (models/mipnerf360/model.py:30-195), vanilla NeRF, the encoder
// and the per-scene pre-projection of the NeO-360 feature maps.
//
// One CTA per 128 x BN output tile: warp 8 = TMA producer (one lane), warps 0-7 = two consumer warpgroups, each owning 64 rows of the
// tile (wgmma m64nBNk16, accumulators in registers).  3-stage shared-memory ring (A 128 x 64, W BN x 64 per stage) with full / empty
// mbarriers; two CTAs fit on an SM, so one CTA's epilogue (bias -> ReLU -> fp16 -> global) overlaps the other's main loop.
//
// Beside it: f32_to_f16_pad (weight / activation packing) and rowdot_f16, the N = 1 / 3 density and rgb heads of the same paths.
#include "common.cuh"
#include "hopper.cuh"
#include <cuda.h>
#include <cuda_fp16.h>

namespace neo {
namespace gemm {
using namespace hopper;

constexpr int BM = 128, BK = 64, kStages = 3, kConsumerWarps = 8, kThreads = (kConsumerWarps + 1) * 32;

template <int BN> struct Acc;
template <> struct Acc<128> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b) { wgmma_ss_n128(d, a, b); }
};
template <> struct Acc<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b) { wgmma_ss_n64(d, a, b); }
};

template <int BN>
__global__ void __launch_bounds__(kThreads, 2)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const float* __restrict__ bias,
                __half* __restrict__ C, long long M, int K, long long ldc, int relu) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
    constexpr uint32_t A_BYTES = BM * BK * 2, W_BYTES = BN * BK * 2, STAGE = A_BYTES + W_BYTES;
    const uint32_t bar0 = sbase + kStages * STAGE;
    auto FULL = [&](int s) { return bar0 + 8u * s; };
    auto EMPTY = [&](int s) { return bar0 + 8u * (kStages + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(FULL(s), 1); mbar_init(EMPTY(s), kConsumerWarps / 4); }
        mbar_init_fence();
    }
    __syncthreads();
    const int kblocks = K / BK;
    const long long m0 = (long long)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;

    if (warp == kConsumerWarps) {
        if (lane == 0) {
            for (int kb = 0; kb < kblocks; ++kb) {
                const uint32_t s = kb % kStages, ph = (kb / kStages) & 1u;
                mbar_wait(EMPTY(s), ph ^ 1u);
                mbar_expect_tx(FULL(s), STAGE);
                tma_load_2d(sbase + s * STAGE, &tmA, kb * BK, (int)m0, FULL(s));
                tma_load_2d(sbase + s * STAGE + A_BYTES, &tmW, kb * BK, n0, FULL(s));
            }
        }
        return;
    }
    const int wg = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < kblocks; ++kb) {
        const uint32_t s = kb % kStages, ph = (kb / kStages) & 1u;
        mbar_wait(FULL(s), ph);
        const uint32_t sa = sbase + s * STAGE + wg * 64 * 128, sw = sbase + s * STAGE + A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < BK / 16; ++ks) Acc<BN>::mma(acc, desc_sw128(sa + ks * 32), desc_sw128(sw + ks * 32));
        wgmma_commit();
        wgmma_wait<1>();                                   // the previous k-block's MMAs are done: its stage goes back to the producer
        if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(EMPTY((kb - 1) % kStages));
    }
    wgmma_wait<0>();
    const int t = lane & 3;
    const long long row0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + 2 * t;
        const float b0 = bias ? __ldg(bias + col) : 0.f, b1 = bias ? __ldg(bias + col + 1) : 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const long long r = row0 + 8 * i;
            float v0 = acc[4 * j + 2 * i] + b0, v1 = acc[4 * j + 2 * i + 1] + b1;
            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (r < M) *reinterpret_cast<__half2*>(C + r * ldc + col) = __floats2half2_rn(v0, v1);
        }
    }
}

// out[r][c] = fp16(in[r][c]) for c < cols_in, 0 for cols_in <= c < cols_out          (weight / activation packing with K padding)
__global__ void f32_to_f16_pad_kernel(const float* __restrict__ in, long long rows, int cols_in, long long ld_in, __half* __restrict__ out,
                                      int cols_out, long long ld_out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * cols_out) return;
    const long long r = idx / cols_out;
    const int c = (int)(idx % cols_out);
    out[r * ld_out + c] = __float2half_rn(c < cols_in ? in[r * ld_in + c] : 0.f);
}

// ---- tiny-N head: out[m][c] = sum_k fp16 h[m][k] * w[c][k] + b[c]  (density: N = 1, rgb: N = 3) ----
// HBM-bound (one pass over the activation rows).  8 lanes per row, 4 rows per warp: every load instruction fetches four whole
// 128-byte lines; the weights sit in shared memory (fp32, read as broadcast float4); 3 shuffles finish a row.
constexpr int kRowdotIters = 4;          // row groups per warp: 8 warps x 4 rows x 4 = 128 rows per block
template <int N>
__global__ void __launch_bounds__(256) rowdot_f16_kernel(const __half* __restrict__ H, long long ld, int K, const float* __restrict__ Wt,
                                                         const float* __restrict__ b, long long M, float* __restrict__ out) {
    extern __shared__ __align__(16) float wsm[];          // [N][K]
    for (int i = threadIdx.x; i < N * K; i += blockDim.x) wsm[i] = Wt[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, sub = lane & 7, rsel = lane >> 3, warp = threadIdx.x >> 5;
    float bias[N];
#pragma unroll
    for (int c = 0; c < N; ++c) bias[c] = b[c];
#pragma unroll 1
    for (int it = 0; it < kRowdotIters; ++it) {
        const long long m = (((long long)blockIdx.x * kRowdotIters + it) * 8 + warp) * 4 + rsel;
        float acc[N];
#pragma unroll
        for (int c = 0; c < N; ++c) acc[c] = 0.f;
        if (m < M) {
            const __half* h = H + m * ld;
            for (int k = sub * 8; k < K; k += 64) {
                const uint4 v = *reinterpret_cast<const uint4*>(h + k);
                const __half2* hv = reinterpret_cast<const __half2*>(&v);
                const float2 f0 = __half22float2(hv[0]), f1 = __half22float2(hv[1]), f2 = __half22float2(hv[2]), f3 = __half22float2(hv[3]);
#pragma unroll
                for (int c = 0; c < N; ++c) {
                    const float4 w0 = *reinterpret_cast<const float4*>(wsm + c * K + k), w1 = *reinterpret_cast<const float4*>(wsm + c * K + k + 4);
                    acc[c] = fmaf(f0.x, w0.x, fmaf(f0.y, w0.y, fmaf(f1.x, w0.z, fmaf(f1.y, w0.w,
                             fmaf(f2.x, w1.x, fmaf(f2.y, w1.y, fmaf(f3.x, w1.z, fmaf(f3.y, w1.w, acc[c]))))))));
                }
            }
        }
#pragma unroll
        for (int c = 0; c < N; ++c) {
            acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], 1);
            acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], 2);
            acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], 4);
        }
        if (m < M && sub == 0) {
#pragma unroll
            for (int c = 0; c < N; ++c) out[m * N + c] = acc[c] + bias[c];
        }
    }
}

static int make_tmap_2d(CUtensorMap* out, const void* base, long long rows, int K, long long ld, int box_rows) {
    typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeTiled encode = nullptr;
    if (!encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qr;
        NEO_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr));
        if (!fn || qr != cudaDriverEntryPointSuccess) { set_error("cuTensorMapEncodeTiled not available from this driver"); return NEO_ERR_UNSUPPORTED; }
        encode = reinterpret_cast<EncodeTiled>(fn);
    }
    const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows}, estr[2] = {1, 1};
    const CUresult r = encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) for a %lld x %d operand (ld %lld)", (int)r, rows, K, ld); return NEO_ERR_CUDA; }
    return NEO_OK;
}

template <int BN>
static int launch(const __half* A, long long lda, const __half* W, long long ldw, const float* bias, __half* C, long long ldc, long long M,
                  int N, int K, int relu, cudaStream_t s) {
    alignas(64) CUtensorMap tmA, tmW;
    int rc;
    if ((rc = make_tmap_2d(&tmA, A, M, K, lda, BM))) return rc;
    if ((rc = make_tmap_2d(&tmW, W, N, K, ldw, BN))) return rc;
    const long long m_tiles = (M + BM - 1) / BM;
    if (m_tiles > 0x7fffffffLL) { set_error("gemm_f16: M = %lld is too large", M); return NEO_ERR_UNSUPPORTED; }
    const size_t smem = (size_t)kStages * (BM * BK * 2 + BN * BK * 2) + 8 * 2 * kStages + 1024;
    NEO_CUDA(cudaFuncSetAttribute(gemm_f16_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gemm_f16_kernel<BN><<<dim3((unsigned)m_tiles, N / BN), kThreads, smem, s>>>(tmA, tmW, bias, C, M, K, ldc, relu);
    NEO_LAUNCH_CHECK("gemm_f16_kernel");
    return NEO_OK;
}

}  // namespace gemm

// C (M x N, row stride ldc) = act(A (M x K, row stride lda) . W (N x K, row stride ldw)^T + bias); fp16 in / out, fp32 accumulate.
// K % 64 == 0, N % 64 == 0, 16-byte aligned rows.  Only columns [0, N) of rows [0, M) of C are written, so A may live in other
// columns of C's own rows (the Mip-NeRF 360 and vanilla NeRF activation buffers keep [h | features] side by side).
int gemm_f16(const void* A, long long lda, const void* W, long long ldw, const float* bias, void* C, long long ldc, long long M, int N, int K,
             int relu, cudaStream_t s) {
    using namespace gemm;
    if (!A || !W || !C) { set_error("gemm_f16: null operand"); return NEO_ERR_INVALID; }
    if (M <= 0 || N <= 0 || K <= 0 || (K % BK) || (N % 64) || (lda % 8) || (ldw % 8) || (ldc % 8) || lda < K || ldw < K || ldc < N) {
        set_error("gemm_f16: need M,N,K > 0, K %% 64 == 0, N %% 64 == 0, row strides %% 8 == 0, lda, ldw >= K and ldc >= N "
                  "(got M=%lld N=%d K=%d lda=%lld ldw=%lld ldc=%lld)", M, N, K, lda, ldw, ldc);
        return NEO_ERR_INVALID;
    }
    if (((uintptr_t)A | (uintptr_t)W | (uintptr_t)C) & 15u) { set_error("gemm_f16: operands must be 16-byte aligned"); return NEO_ERR_INVALID; }
    const __half *a = (const __half*)A, *w = (const __half*)W;
    __half* c = (__half*)C;
    if (N % 128 == 0) return launch<128>(a, lda, w, ldw, bias, c, ldc, M, N, K, relu, s);
    return launch<64>(a, lda, w, ldw, bias, c, ldc, M, N, K, relu, s);
}
int f32_to_f16_pad(const float* in, long long rows, int cols_in, long long ld_in, void* out, int cols_out, long long ld_out, cudaStream_t s) {
    const long long total = rows * cols_out;
    if (total <= 0) return NEO_OK;
    gemm::f32_to_f16_pad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(in, rows, cols_in, ld_in, (__half*)out, cols_out, ld_out);
    NEO_LAUNCH_CHECK("f32_to_f16_pad_kernel");
    return NEO_OK;
}
// out (M x N) fp32 = H (M x K, fp16, row stride ld) . W (N x K, fp32)^T + b: the density / rgb heads of the vanilla NeRF, Mip-NeRF 360 and
// encoder tensor-core paths.
int launch_rowdot_f16(const void* H, long long ld, int K, const float* W, const float* b, int N, long long M, float* out, cudaStream_t s) {
    if (M <= 0) return NEO_OK;
    if ((K % 8) || (ld % 8) || (N != 1 && N != 3)) { set_error("rowdot_f16: K %% 8, ld %% 8 and N in {1, 3} required (K=%d ld=%lld N=%d)", K, ld, N); return NEO_ERR_INVALID; }
    if (K <= 0 || ld < K || (size_t)N * K * sizeof(float) > 48 * 1024) { set_error("rowdot_f16: need 0 < K <= ld and N*K*4 <= 48 KB (K=%d ld=%lld N=%d)", K, ld, N); return NEO_ERR_INVALID; }
    if (!H || !W || !b || !out || (reinterpret_cast<uintptr_t>(H) & 15)) { set_error("rowdot_f16: null pointer or H not 16-byte aligned"); return NEO_ERR_INVALID; }
    const unsigned grid = (unsigned)((M + 8 * 4 * gemm::kRowdotIters - 1) / (8 * 4 * gemm::kRowdotIters));
    const size_t smem = (size_t)N * K * sizeof(float);
    if (N == 1) gemm::rowdot_f16_kernel<1><<<grid, 256, smem, s>>>((const __half*)H, ld, K, W, b, M, out);
    else gemm::rowdot_f16_kernel<3><<<grid, 256, smem, s>>>((const __half*)H, ld, K, W, b, M, out);
    NEO_LAUNCH_CHECK("rowdot_f16_kernel");
    return NEO_OK;
}

}  // namespace neo

// Stage-level entry point of gemm_f16 itself, at the strides and aliasing its callers use: fp16 device operands, asynchronous on `stream`.
extern "C" int neo_tc_gemm_f16(const void* A, long long lda, const void* W, long long ldw, const float* bias, void* C, long long ldc, long long M,
                               int N, int K, int relu, void* stream) {
    return neo::gemm_f16(A, lda, W, ldw, bias, C, ldc, M, N, K, relu, (cudaStream_t)stream);
}
// Stage-level entry point of rowdot_f16, the tiny-N head of the vanilla NeRF, Mip-NeRF 360 and encoder paths.
extern "C" int neo_tc_rowdot_f16(const void* H, long long ld, int K, const float* W, const float* b, int N, long long M, float* out, void* stream) {
    return neo::launch_rowdot_f16(H, ld, K, W, b, N, M, out, (cudaStream_t)stream);
}
