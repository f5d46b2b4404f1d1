// gemm_simt.cuh -- exact fp32 GEMM  C[M,N] = A[M,K] (fp32) x W[N,K]^T (fp16 weights) on the CUDA cores.
// This is the arithmetic-exact path (every product and sum in fp32, like the reference's Candle F32
// Linear::forward, src/models/common/modules.rs:81-87,538-577).  It is the validation
// baseline for the wgmma split-fp16 kernel in gemm_tc.cuh and the fallback for shapes that kernel
// does not tile (tiny test configs).
#pragma once
#include "common.cuh"

namespace aha {

enum GemmEpi {
    EPI_STORE = 0,   // C = acc (+bias)
    EPI_RESID = 1,   // C = resid + acc (+bias)      (resid may alias C)
    EPI_ACT = 2,     // C = act(acc + bias)
    EPI_SWIGLU = 3,  // C[m, c/2] = silu(acc[m,c]) * acc[m,c+1]  (gate/up rows interleaved), ldc = N/2
};

struct GemmArgs {
    const float* A; int lda;
    const __half* W;          // [N, K] row-major
    const float* bias;        // [N] or nullptr
    const float* resid; int ldr;
    float* C; int ldc;
    int M, N, K;
    int act;
    // LoRA tail (lora.cuh): K2 more columns of the sum, A2 [M][K2] (fp32, ld lda2) times W2 [N][K2], after the K base columns
    const float* A2 = nullptr; int lda2 = 0;
    const __half* W2 = nullptr; int K2 = 0;
};

template <int EPI>
__global__ void __launch_bounds__(256) gemm_simt_kernel(GemmArgs g) {
    constexpr int BM = 128, BN = 128, BK = 16, PAD = 4;
    __shared__ __align__(16) float As[2][BK][BM + PAD];
    __shared__ __align__(16) float Bs[2][BK][BN + PAD];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

    // global->register staging
    const int a_row = tid >> 2;         // 0..63 (+64)
    const int a_k = (tid & 3) * 4;      // 0,4,8,12
    const int b_row = tid >> 1;         // 0..127
    const int b_k = (tid & 1) * 8;      // 0,8
    float4 ra[2];
    uint4 rb;

    auto load_tiles = [&](int k0) {
        const bool tail = k0 >= g.K;
        const float* A = tail ? g.A2 : g.A;
        const __half* W = tail ? g.W2 : g.W;
        const int lda = tail ? g.lda2 : g.lda, ldw = tail ? g.K2 : g.K, k = tail ? k0 - g.K : k0;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            int m = m0 + a_row + i * 64;
            ra[i] = (m < g.M) ? *reinterpret_cast<const float4*>(A + (size_t)m * lda + k + a_k)
                              : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        int n = n0 + b_row;
        rb = (n < g.N) ? *reinterpret_cast<const uint4*>(W + (size_t)n * ldw + k + b_k) : make_uint4(0, 0, 0, 0);
    };
    auto store_tiles = [&](int buf) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            int r = a_row + i * 64;
            As[buf][a_k + 0][r] = ra[i].x; As[buf][a_k + 1][r] = ra[i].y;
            As[buf][a_k + 2][r] = ra[i].z; As[buf][a_k + 3][r] = ra[i].w;
        }
        float2 f0 = h2_to_f2(rb.x), f1 = h2_to_f2(rb.y), f2 = h2_to_f2(rb.z), f3 = h2_to_f2(rb.w);
        Bs[buf][b_k + 0][b_row] = f0.x; Bs[buf][b_k + 1][b_row] = f0.y;
        Bs[buf][b_k + 2][b_row] = f1.x; Bs[buf][b_k + 3][b_row] = f1.y;
        Bs[buf][b_k + 4][b_row] = f2.x; Bs[buf][b_k + 5][b_row] = f2.y;
        Bs[buf][b_k + 6][b_row] = f3.x; Bs[buf][b_k + 7][b_row] = f3.y;
    };

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    const int nk = (g.K + g.K2) / BK;
    load_tiles(0);
    store_tiles(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) load_tiles((kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
            float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nk) {
            store_tiles(buf ^ 1);
            __syncthreads();
        }
    }

    // epilogue
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (m >= g.M) continue;
#pragma unroll
        for (int jh = 0; jh < 2; ++jh) {
            const int n = n0 + (jh == 0 ? tx * 4 : 64 + tx * 4);
            if (n >= g.N) continue;  // N % 4 == 0 is required by the host wrapper
            float v[4] = {acc[i][jh * 4 + 0], acc[i][jh * 4 + 1], acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]};
            if (g.bias) {
#pragma unroll
                for (int j = 0; j < 4; ++j) v[j] += g.bias[n + j];
            }
            if (EPI == EPI_SWIGLU) {
                float2 o = make_float2(silu_f(v[0]) * v[1], silu_f(v[2]) * v[3]);
                *reinterpret_cast<float2*>(g.C + (size_t)m * g.ldc + n / 2) = o;
            } else {
                if (EPI == EPI_ACT) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) v[j] = apply_act(g.act, v[j]);
                }
                if (EPI == EPI_RESID) {
                    float4 r = *reinterpret_cast<const float4*>(g.resid + (size_t)m * g.ldr + n);
                    v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
                }
                *reinterpret_cast<float4*>(g.C + (size_t)m * g.ldc + n) = make_float4(v[0], v[1], v[2], v[3]);
            }
        }
    }
}

inline void gemm_simt(cudaStream_t st, int epi, const GemmArgs& g) {
    AHA_REQUIRE(g.K % 16 == 0 && g.K2 % 16 == 0, "gemm_simt: K must be a multiple of 16");
    AHA_REQUIRE(g.K2 == 0 || (g.A2 && g.W2 && g.lda2 % 4 == 0), "gemm_simt: the tail needs A2 / W2");
    AHA_REQUIRE(g.N % 4 == 0 && g.lda % 4 == 0 && g.ldc % 2 == 0, "gemm_simt: N/lda alignment");
    if (g.M == 0) return;
    dim3 grid(ceil_div(g.N, 128), ceil_div(g.M, 128));
    switch (epi) {
        case EPI_STORE: gemm_simt_kernel<EPI_STORE><<<grid, 256, 0, st>>>(g); break;
        case EPI_RESID: gemm_simt_kernel<EPI_RESID><<<grid, 256, 0, st>>>(g); break;
        case EPI_ACT: gemm_simt_kernel<EPI_ACT><<<grid, 256, 0, st>>>(g); break;
        case EPI_SWIGLU: gemm_simt_kernel<EPI_SWIGLU><<<grid, 256, 0, st>>>(g); break;
        default: AHA_REQUIRE(false, "gemm_simt: bad epilogue");
    }
    AHA_CUDA_CHECK(cudaGetLastError());
}

}  // namespace aha
