// Generic dense layer on Hopper tensor cores (sm_90a):  C[M][N] = act(A[M][K] . W[N][K]^T + bias)   fp16 operands, fp32 accumulate.
// A and W are K-major (row-major activations, nn.Linear weights), so both operands are staged by 2-D TMA tile loads
// (cp.async.bulk.tensor.2d, 128-byte swizzle) straight into the layout wgmma reads.  Used by the tensor-core paths of the wide
// MLPs: Mip-NeRF 360's 8 x 1024 NeRF MLP and 4 x 256 proposal MLPs (models/mipnerf360/model.py:30-195), vanilla NeRF, the encoder
// and the per-scene pre-projection of the NeO-360 feature maps.
//
// One CTA per 128 x BN output tile: warp 8 = TMA producer (one lane), warps 0-7 = two consumer warpgroups, each owning 64 rows of the
// tile (wgmma m64nBNk16, accumulators in registers).  3-stage shared-memory ring (A 128 x 64, W BN x 64 per stage) with full / empty
// mbarriers; two CTAs fit on an SM, so one CTA's epilogue (bias -> ReLU -> fp16 -> global) overlaps the other's main loop.
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

}  // namespace neo

// Stage-level entry point (self-test / parity test of the tensor-core dense layer): A (M,K), W (N,K) fp32 device -> out (M,N) fp32 =
// act(fp16(A) . fp16(W)^T + bias) rounded to fp16, computed by gemm_f16_kernel.  K % 64 == 0, N % 64 == 0.
extern "C" int neo_tc_dense(const float* A, const float* W, const float* bias, long long M, int N, int K, int relu, float* out, void* stream);

namespace neo { namespace gemm {
__global__ void f16_to_f32_kernel(const __half* __restrict__ in, long long n, float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = __half2float(in[i]);
}
} }

extern "C" int neo_tc_dense(const float* A, const float* W, const float* bias, long long M, int N, int K, int relu, float* out, void* stream) {
    using namespace neo;
    if (!A || !W || !out || M <= 0) { set_error("neo_tc_dense: bad arguments"); return NEO_ERR_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    __half *a = nullptr, *w = nullptr, *c = nullptr;
    NEO_CUDA(cudaMalloc(&a, (size_t)M * K * 2));
    NEO_CUDA(cudaMalloc(&w, (size_t)N * K * 2));
    NEO_CUDA(cudaMalloc(&c, (size_t)M * N * 2));
    int rc = f32_to_f16_pad(A, M, K, K, a, K, K, s);
    if (!rc) rc = f32_to_f16_pad(W, N, K, K, w, K, K, s);
    if (!rc) rc = gemm_f16(a, K, w, K, bias, c, N, M, N, K, relu, s);
    if (!rc) {
        gemm::f16_to_f32_kernel<<<(unsigned)(((long long)M * N + 255) / 256), 256, 0, s>>>(c, (long long)M * N, out);
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) rc = cuda_fail(e, "neo_tc_dense");
    }
    cudaFree(a); cudaFree(w); cudaFree(c);
    return rc;
}

// Stage-level entry point of gemm_f16 itself, at the strides and aliasing its callers use: fp16 device operands, asynchronous on `stream`.
extern "C" int neo_tc_gemm_f16(const void* A, long long lda, const void* W, long long ldw, const float* bias, void* C, long long ldc, long long M,
                               int N, int K, int relu, void* stream) {
    return neo::gemm_f16(A, lda, W, ldw, bias, C, ldc, M, N, K, relu, (cudaStream_t)stream);
}
