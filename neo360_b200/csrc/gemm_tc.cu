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
#include <cuda_bf16.h>
#include <type_traits>

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

template <int BN> struct AccBf16;
template <> struct AccBf16<128> {
    template <int T> static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b) { wgmma_ss_n128_bf16<T, T>(d, a, b); }
};
template <> struct AccBf16<64> {
    template <int T> static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b) { wgmma_ss_n64_bf16<T, T>(d, a, b); }
};

// The one TMA / wgmma main loop of every product form: acc (this thread's fragment of the 128 x BN tile at (m0, n0)) = sum over k-blocks
// of split blockIdx.z (of `splits`: a fixed share of the `kblocks` k-blocks) of A . W^T, with m0 = blockIdx.x BM, n0 = blockIdx.y BN.  K-major (MN = false): A (rows m, 64-column k-blocks) and W (rows n) are nn.Linear-style operands, one TMA box
// each per stage.  MN-major (MN = true, bf16 only): A and W are both row-major over the reduction axis (A^T . W, the weight gradient):
// a stage holds 64 reduction rows as boxes of 64 columns, two for A (128 m) and BN / 64 for W.  Returns false in the producer warp.
template <typename T, int BN, bool MN>
__device__ __forceinline__ bool gemm_mainloop(const CUtensorMap* tmA, const CUtensorMap* tmW, int kblocks, int splits, long long& m0, int& n0,
                                              float (&acc)[BN / 2]) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
    constexpr uint32_t A_BYTES = BM * BK * 2, W_BYTES = BN * BK * 2, STAGE = A_BYTES + W_BYTES, BOX = 64 * BK * 2;
    const uint32_t bar0 = sbase + kStages * STAGE;
    auto FULL = [&](int s) { return bar0 + 8u * s; };
    auto EMPTY = [&](int s) { return bar0 + 8u * (kStages + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(FULL(s), 1); mbar_init(EMPTY(s), kConsumerWarps / 4); }
        mbar_init_fence();
    }
    __syncthreads();
    const int kb0 = splits == 1 ? 0 : (int)((long long)kblocks * blockIdx.z / splits);
    const int kb1 = splits == 1 ? kblocks : (int)((long long)kblocks * (blockIdx.z + 1) / splits);
    m0 = (long long)blockIdx.x * BM;
    n0 = blockIdx.y * BN;

    if (warp == kConsumerWarps) {
        if (lane == 0) {
            for (int kb = kb0; kb < kb1; ++kb) {
                const uint32_t s = (kb - kb0) % kStages, ph = ((kb - kb0) / kStages) & 1u;
                mbar_wait(EMPTY(s), ph ^ 1u);
                mbar_expect_tx(FULL(s), STAGE);
                if constexpr (MN) {
#pragma unroll
                    for (int c = 0; c < BM / 64; ++c) tma_load_2d(sbase + s * STAGE + c * BOX, tmA, (int)m0 + 64 * c, kb * BK, FULL(s));
#pragma unroll
                    for (int c = 0; c < BN / 64; ++c) tma_load_2d(sbase + s * STAGE + A_BYTES + c * BOX, tmW, n0 + 64 * c, kb * BK, FULL(s));
                } else {
                    tma_load_2d(sbase + s * STAGE, tmA, kb * BK, (int)m0, FULL(s));
                    tma_load_2d(sbase + s * STAGE + A_BYTES, tmW, kb * BK, n0, FULL(s));
                }
            }
        }
        return false;
    }
    const int wg = warp >> 2;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int i = 0; i < kb1 - kb0; ++i) {                  // counted from 0: a split's accumulators stay wgmma-only inside the loop
        const uint32_t s = i % kStages, ph = (i / kStages) & 1u;
        mbar_wait(FULL(s), ph);
        const uint32_t sa = sbase + s * STAGE + wg * 64 * 128, sw = sbase + s * STAGE + A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < BK / 16; ++ks) {
            if constexpr (MN) AccBf16<BN>::template mma<1>(acc, desc_sw128_mn(sa + ks * 2048, BOX), desc_sw128_mn(sw + ks * 2048, BOX));
            else if constexpr (std::is_same<T, __half>::value) Acc<BN>::mma(acc, desc_sw128(sa + ks * 32), desc_sw128(sw + ks * 32));
            else AccBf16<BN>::template mma<0>(acc, desc_sw128(sa + ks * 32), desc_sw128(sw + ks * 32));
        }
        wgmma_commit();
        wgmma_wait<1>();                                   // the previous k-block's MMAs are done: its stage goes back to the producer
        if (i > 0 && (threadIdx.x & 127) == 0) mbar_arrive(EMPTY((i - 1) % kStages));
    }
    wgmma_wait<0>();
    return true;
}

template <int BN>
__global__ void __launch_bounds__(kThreads, 2)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const float* __restrict__ bias,
                __half* __restrict__ C, long long M, int K, long long ldc, int relu) {
    long long m0;
    int n0;
    float acc[BN / 2];
    if (!gemm_mainloop<__half, BN, false>(&tmA, &tmW, K / BK, 1, m0, n0, acc)) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
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

// Training forms (bf16 operands, fp32 accumulation; csrc/dense_train.cu): the forward epilogues bias + ReLU -> bf16, bias -> bf16 and
// no bias -> fp32 (also the weight gradient's per-split partial, at C + blockIdx.z zstride); the data gradient's epilogue adds the rank-1 term
// g_sig[r] w_sig[c] and applies the ReLU mask [X[r][c] > 0] of the saved bf16 layer input before rounding to bf16.
enum Epi { kEpiReluBf16 = 0, kEpiBf16 = 1, kEpiF32 = 2, kEpiDgrad = 3 };
struct EpiParams {
    const float* bias;
    void* C;
    long long ldc, M, zstride;                    // rows r < M of C are written
    const __nv_bfloat16* X;                       // dgrad: ReLU mask source (NULL: no mask), row stride ldx
    long long ldx;
    const float *g_sig, *w_sig;                   // dgrad: rank-1 addend (NULL: none)
    int kblocks, splits;
};

template <int BN, int EPI, bool MN>
__global__ void __launch_bounds__(kThreads, 2)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const __grid_constant__ EpiParams P) {
    long long m0;
    int n0;
    float acc[BN / 2];
    if (!gemm_mainloop<__nv_bfloat16, BN, MN>(&tmA, &tmW, P.kblocks, MN ? P.splits : 1, m0, n0, acc)) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    const int t = lane & 3;
    const long long row0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    float* const Cf = (float*)P.C + blockIdx.z * P.zstride;
    __nv_bfloat16* const Cb = (__nv_bfloat16*)P.C;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + 2 * t;
        constexpr bool has_bias = EPI == kEpiReluBf16 || EPI == kEpiBf16;
        const float b0 = has_bias && P.bias ? __ldg(P.bias + col) : 0.f, b1 = has_bias && P.bias ? __ldg(P.bias + col + 1) : 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const long long r = row0 + 8 * i;
            float v0 = acc[4 * j + 2 * i] + b0, v1 = acc[4 * j + 2 * i + 1] + b1;
            if constexpr (EPI == kEpiReluBf16) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (r >= P.M) continue;
            if constexpr (EPI == kEpiDgrad) {
                if (P.g_sig) { const float g = __ldg(P.g_sig + r); v0 = fmaf(g, __ldg(P.w_sig + col), v0); v1 = fmaf(g, __ldg(P.w_sig + col + 1), v1); }
                if (P.X) {
                    const float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(P.X + r * P.ldx + col));
                    v0 = x.x > 0.f ? v0 : 0.f;
                    v1 = x.y > 0.f ? v1 : 0.f;
                }
            }
            if constexpr (EPI == kEpiF32) *reinterpret_cast<float2*>(Cf + r * P.ldc + col) = make_float2(v0, v1);
            else *reinterpret_cast<__nv_bfloat162*>(Cb + r * P.ldc + col) = __floats2bfloat162_rn(v0, v1);
        }
    }
}

template <typename T> __device__ __forceinline__ T from_f32(float x);
template <> __device__ __forceinline__ __half from_f32<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }
__device__ __forceinline__ float2 to_f32x2(__half2 h) { return __half22float2(h); }
__device__ __forceinline__ float2 to_f32x2(__nv_bfloat162 h) { return __bfloat1622float2(h); }
template <typename T> struct Pair;
template <> struct Pair<__half> { using type = __half2; };
template <> struct Pair<__nv_bfloat16> { using type = __nv_bfloat162; };

// out[r][c] = T(in[r][c]) for c < cols_in, 0 for cols_in <= c < cols_out          (weight / activation packing with K padding)
template <typename T>
__global__ void f32_to_f16_pad_kernel(const float* __restrict__ in, long long rows, int cols_in, long long ld_in, T* __restrict__ out,
                                      int cols_out, long long ld_out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * cols_out) return;
    const long long r = idx / cols_out;
    const int c = (int)(idx % cols_out);
    out[r * ld_out + c] = from_f32<T>(c < cols_in ? in[r * ld_in + c] : 0.f);
}

// ---- tiny-N head: out[m][c] = sum_k h[m][k] * w[c][k] + b[c], h fp16 or bf16  (density: N = 1, rgb: N = 3) ----
// HBM-bound (one pass over the activation rows).  8 lanes per row, 4 rows per warp: every load instruction fetches four whole
// 128-byte lines; the weights sit in shared memory (fp32, read as broadcast float4); 3 shuffles finish a row.
constexpr int kRowdotIters = 4;          // row groups per warp: 8 warps x 4 rows x 4 = 128 rows per block
template <int N, typename T>
__global__ void __launch_bounds__(256) rowdot_f16_kernel(const T* __restrict__ H, long long ld, int K, const float* __restrict__ Wt,
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
            const T* h = H + m * ld;
            for (int k = sub * 8; k < K; k += 64) {
                const uint4 v = *reinterpret_cast<const uint4*>(h + k);
                const typename Pair<T>::type* hv = reinterpret_cast<const typename Pair<T>::type*>(&v);
                const float2 f0 = to_f32x2(hv[0]), f1 = to_f32x2(hv[1]), f2 = to_f32x2(hv[2]), f3 = to_f32x2(hv[3]);
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

static int make_tmap_2d(CUtensorMap* out, const void* base, long long rows, int K, long long ld, int box_rows,
                        CUtensorMapDataType type = CU_TENSOR_MAP_DATA_TYPE_FLOAT16) {
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
    const CUresult r = encode(out, type, 2, const_cast<void*>(base), dims, strides, box, estr,
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

template <int BN, int EPI, bool MN>
static int launch_bf16(const CUtensorMap& tmA, const CUtensorMap& tmW, const EpiParams& P, long long m_tiles, int n_tiles, cudaStream_t s) {
    if (m_tiles > 0x7fffffffLL) { set_error("gemm_bf16: %lld row tiles is too many", m_tiles); return NEO_ERR_UNSUPPORTED; }
    const size_t smem = (size_t)kStages * (BM * BK * 2 + BN * BK * 2) + 8 * 2 * kStages + 1024;
    NEO_CUDA(cudaFuncSetAttribute(gemm_bf16_kernel<BN, EPI, MN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gemm_bf16_kernel<BN, EPI, MN><<<dim3((unsigned)m_tiles, n_tiles, P.splits), kThreads, smem, s>>>(tmA, tmW, P);
    NEO_LAUNCH_CHECK("gemm_bf16_kernel");
    return NEO_OK;
}

// K-major product forms (forward, dgrad): A (M, K), W (N, K) bf16
template <int EPI>
static int launch_kmajor_bf16(const void* A, long long lda, const void* W, long long ldw, long long M, int N, int K, EpiParams P, cudaStream_t s) {
    alignas(64) CUtensorMap tmA, tmW;
    const int bn = N % 128 == 0 ? 128 : 64;
    int rc;
    if ((rc = make_tmap_2d(&tmA, A, M, K, lda, BM, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16))) return rc;
    if ((rc = make_tmap_2d(&tmW, W, N, K, ldw, bn, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16))) return rc;
    P.M = M; P.zstride = 0; P.kblocks = K / BK; P.splits = 1;
    const long long m_tiles = (M + BM - 1) / BM;
    return bn == 128 ? launch_bf16<128, EPI, false>(tmA, tmW, P, m_tiles, N / 128, s) : launch_bf16<64, EPI, false>(tmA, tmW, P, m_tiles, N / 64, s);
}

static bool kmajor_ok(const char* who, const void* A, long long lda, const void* W, long long ldw, const void* C, long long ldc, long long M,
                      int N, int K) {
    if (!A || !W || !C) { set_error("%s: null operand", who); return false; }
    if (M <= 0 || N <= 0 || K <= 0 || (K % BK) || (N % 64) || (lda % 8) || (ldw % 8) || (ldc % 8) || lda < K || ldw < K || ldc < N) {
        set_error("%s: need M,N,K > 0, K %% 64 == 0, N %% 64 == 0, row strides %% 8 == 0, lda, ldw >= K and ldc >= N "
                  "(got M=%lld N=%d K=%d lda=%lld ldw=%lld ldc=%lld)", who, M, N, K, lda, ldw, ldc);
        return false;
    }
    if (((uintptr_t)A | (uintptr_t)W | (uintptr_t)C) & 15u) { set_error("%s: operands must be 16-byte aligned", who); return false; }
    return true;
}

}  // namespace gemm

// Training forms, bf16 operands and fp32 accumulation, same shape rules as gemm_f16.  C (M x N) = A . W^T + bias, then ReLU -> bf16
// (epi 0), -> bf16 (1) or -> fp32 (2).
int gemm_bf16(const void* A, long long lda, const void* W, long long ldw, const float* bias, void* C, long long ldc, long long M, int N, int K,
              int epi, cudaStream_t s) {
    using namespace gemm;
    if (!kmajor_ok("gemm_bf16", A, lda, W, ldw, C, ldc, M, N, K)) return NEO_ERR_INVALID;
    if (epi < kEpiReluBf16 || epi > kEpiF32) { set_error("gemm_bf16: epilogue %d, must be 0, 1 or 2", epi); return NEO_ERR_INVALID; }
    EpiParams P = {};
    P.bias = bias; P.C = C; P.ldc = ldc;
    if (epi == kEpiReluBf16) return launch_kmajor_bf16<kEpiReluBf16>(A, lda, W, ldw, M, N, K, P, s);
    if (epi == kEpiBf16) return launch_kmajor_bf16<kEpiBf16>(A, lda, W, ldw, M, N, K, P, s);
    return launch_kmajor_bf16<kEpiF32>(A, lda, W, ldw, M, N, K, P, s);
}
// dX (M x N, bf16) = (dY (M x K) . Wt (N x K)^T + g_sig w_sig^T) [X > 0]: the data gradient through a layer whose weight W (K x N) is
// given transposed; X (M x N, row stride ldx, bf16) is the saved layer input (NULL: no mask), g_sig (M) / w_sig (N) fp32 or both NULL.
int dgrad_bf16(const void* dY, long long ldy, const void* Wt, long long ldwt, const void* X, long long ldx, const float* g_sig,
               const float* w_sig, void* dX, long long lddx, long long M, int N, int K, cudaStream_t s) {
    using namespace gemm;
    if (!kmajor_ok("dgrad_bf16", dY, ldy, Wt, ldwt, dX, lddx, M, N, K)) return NEO_ERR_INVALID;
    if ((g_sig == nullptr) != (w_sig == nullptr)) { set_error("dgrad_bf16: g_sig and w_sig must both be given or both be NULL"); return NEO_ERR_INVALID; }
    if (X && (ldx < N || (ldx % 2) || ((uintptr_t)X & 3u))) { set_error("dgrad_bf16: mask rows need ldx >= N, ldx even and 4-byte alignment"); return NEO_ERR_INVALID; }
    EpiParams P = {};
    P.C = dX; P.ldc = lddx; P.X = (const __nv_bfloat16*)X; P.ldx = ldx; P.g_sig = g_sig; P.w_sig = w_sig;
    return launch_kmajor_bf16<kEpiDgrad>(dY, ldy, Wt, ldwt, M, N, K, P, s);
}
// part[z] (N x K, fp32) = sum over the rows of split z of dY (M x N)^T X (M x K), both bf16 and row-major over the M rows, as MN-major
// wgmma operands; split z covers 64-row blocks [nb z / splits, nb (z + 1) / splits), nb = ceil(M / 64) (TMA fills rows past M with zeros).
// Arguments are checked by the caller (dense_train.cu).
int wgrad_bf16_partials(const void* dY, long long ldy, const void* X, long long ldx, long long M, int N, int K, int splits, float* part,
                        cudaStream_t s) {
    using namespace gemm;
    alignas(64) CUtensorMap tmA, tmW;
    const int bn = K % 128 == 0 ? 128 : 64;
    int rc;
    if ((rc = make_tmap_2d(&tmA, dY, M, N, ldy, 64, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16))) return rc;
    if ((rc = make_tmap_2d(&tmW, X, M, K, ldx, 64, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16))) return rc;
    EpiParams P = {};
    P.C = part; P.ldc = K; P.M = N; P.zstride = (long long)N * K; P.kblocks = (int)((M + BK - 1) / BK); P.splits = splits;
    const long long m_tiles = (N + BM - 1) / BM;
    return bn == 128 ? launch_bf16<128, kEpiF32, true>(tmA, tmW, P, m_tiles, K / 128, s) : launch_bf16<64, kEpiF32, true>(tmA, tmW, P, m_tiles, K / 64, s);
}

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
int f32_to_f16_pad(const float* in, long long rows, int cols_in, long long ld_in, void* out, int cols_out, long long ld_out, cudaStream_t s,
                   int bf16) {
    const long long total = rows * cols_out;
    if (total <= 0) return NEO_OK;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (bf16) gemm::f32_to_f16_pad_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(in, rows, cols_in, ld_in, (__nv_bfloat16*)out, cols_out, ld_out);
    else gemm::f32_to_f16_pad_kernel<__half><<<grid, 256, 0, s>>>(in, rows, cols_in, ld_in, (__half*)out, cols_out, ld_out);
    NEO_LAUNCH_CHECK("f32_to_f16_pad_kernel");
    return NEO_OK;
}
// out (M x N) fp32 = H (M x K, fp16 or, with bf16 = 1, bf16; row stride ld) . W (N x K, fp32)^T + b: the density / rgb heads of the vanilla
// NeRF, Mip-NeRF 360 and encoder tensor-core paths, and the density head of their training form.
int launch_rowdot_f16(const void* H, long long ld, int K, const float* W, const float* b, int N, long long M, float* out, cudaStream_t s,
                      int bf16) {
    const char* who = bf16 ? "rowdot_bf16" : "rowdot_f16";
    if (M <= 0) return NEO_OK;
    if ((K % 8) || (ld % 8) || (N != 1 && N != 3)) { set_error("%s: K %% 8, ld %% 8 and N in {1, 3} required (K=%d ld=%lld N=%d)", who, K, ld, N); return NEO_ERR_INVALID; }
    if (K <= 0 || ld < K || (size_t)N * K * sizeof(float) > 48 * 1024) { set_error("%s: need 0 < K <= ld and N*K*4 <= 48 KB (K=%d ld=%lld N=%d)", who, K, ld, N); return NEO_ERR_INVALID; }
    if (!H || !W || !b || !out || (reinterpret_cast<uintptr_t>(H) & 15)) { set_error("%s: null pointer or H not 16-byte aligned", who); return NEO_ERR_INVALID; }
    const unsigned grid = (unsigned)((M + 8 * 4 * gemm::kRowdotIters - 1) / (8 * 4 * gemm::kRowdotIters));
    const size_t smem = (size_t)N * K * sizeof(float);
    if (bf16) {
        if (N == 1) gemm::rowdot_f16_kernel<1, __nv_bfloat16><<<grid, 256, smem, s>>>((const __nv_bfloat16*)H, ld, K, W, b, M, out);
        else gemm::rowdot_f16_kernel<3, __nv_bfloat16><<<grid, 256, smem, s>>>((const __nv_bfloat16*)H, ld, K, W, b, M, out);
    } else if (N == 1) gemm::rowdot_f16_kernel<1, __half><<<grid, 256, smem, s>>>((const __half*)H, ld, K, W, b, M, out);
    else gemm::rowdot_f16_kernel<3, __half><<<grid, 256, smem, s>>>((const __half*)H, ld, K, W, b, M, out);
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
