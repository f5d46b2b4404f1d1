// lora.cuh -- LoRA adapters of a wide batch session as extra k-blocks of the projections they target.
//
// An adapter adds s * B (A x) to a projection y = W x.  Written as one product, y = [W | B_pool] . [x ; t], the update is more K: t is the
// row's shrink output s * A x, and B_pool holds the B columns of every loaded adapter.  So the wgmma kernels that stream W
// (gemv_wide.cuh, gemm_tc.cuh) and the SIMT twin (gemm_simt.cuh) run the update as tail k-blocks after their base k-blocks, and their
// bias / residual / SwiGLU epilogues see the full sum unchanged.
//
// Layout, per layer and per projection group g (qkv, o, gate/up, down):
//   * adapter a owns pool columns [off_g(a), off_g(a) + w_g(a)), off_g(a) a multiple of 16: one sub-block of r columns per target of the
//     group it has in any layer (q, k, v / gate, up in that order), w_g = round16(targets x r);
//   * A_pool [Rp_g][K]: row off_g(a) + j is row j of the adapter's stacked A's (zero rows pad the block and stand for absent targets);
//   * B_pool [N][Rp_g]: the adapter's B's in the base row layout -- q / k / v rows each on their own sub-block (block diagonal), gate and up
//     rows interleaved like TextLayer::gu, each on its own sub-block;
//   * Rp_g is a multiple of the 64-column k-block.
// lora_shrink_kernel writes t [rows][Rp_g]: s * A_pool[c] . x for the columns c of the row's adapter, zero everywhere else.  A k16 slice
// of the tail then belongs to one adapter, and a row adds exact zeros outside its own slices, in the same order whatever else runs.  So a
// row's sum depends only on its own adapter (base rows: on nothing but the base weights), whichever adapters share the step or the pack.
// The tail streams only the k-blocks that hold columns of adapters in use: a device list [count, kb0, kb1, ...] per group.
#pragma once
#include <cuda_fp16.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace aha {

enum LoraGroup { LORA_QKV = 0, LORA_O = 1, LORA_GU = 2, LORA_DOWN = 3, kLoraGroups = 4 };
constexpr int kLoraMaxRank = 64;
constexpr int kLoraAlign = 16;     // an adapter's columns start on a wgmma k16 slice
constexpr int kLoraKb = 64;        // the tail's k-block (kTcBK)

struct LoraTab {                   // one loaded adapter as the shrink kernel sees it
    int off[kLoraGroups];
    int w[kLoraGroups];
    float scale;
};

// The tail of one projection: t (fp16 hi + lo halves, and fp32 for the SIMT twin) [rows][Rp], B_pool [N][Rp] and the device list of the
// k-blocks to stream.  Rp == 0: no tail.
struct LoraTail {
    const __half* t_hi = nullptr;
    const __half* t_lo = nullptr;
    const float* t_f32 = nullptr;
    const __half* B = nullptr;
    int Rp = 0;
    const int* list = nullptr;     // device [1 + Rp / 64]: count, then k-block indices in ascending order
};

// t[j] = s * A_pool . x_j over the columns of row j's adapter, zero elsewhere.  x_j: hi + lo halves (x_hi set) or fp32 (x_f32).  Row j's
// adapter: ad[act ? act[j] : j] (an index into tab, < 0: none).  One CTA per row; warp w takes columns w, w + 8, ... of the adapter, each
// dot product in a fixed lane order and shuffle tree.
__global__ void __launch_bounds__(256) lora_shrink_kernel(const __half* __restrict__ x_hi, const __half* __restrict__ x_lo,
                                                          const float* __restrict__ x_f32, int ldx, int K, const __half* __restrict__ A, int Rp,
                                                          const LoraTab* __restrict__ tab, int g, const int* __restrict__ ad,
                                                          const int* __restrict__ act, __half* __restrict__ t_hi, __half* __restrict__ t_lo,
                                                          float* __restrict__ t_f32) {
    const int j = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int a = ad[act ? act[j] : j];
    int off = 0, w = 0;
    float s = 0.f;
    if (a >= 0) { off = tab[a].off[g]; w = tab[a].w[g]; s = tab[a].scale; }
    const size_t row = (size_t)j * Rp;
    for (int c = tid; c < Rp; c += 256) {
        if (c >= off && c < off + w) continue;
        t_hi[row + c] = __float2half_rn(0.f);
        t_lo[row + c] = __float2half_rn(0.f);
        if (t_f32) t_f32[row + c] = 0.f;
    }
    const size_t xr = (size_t)j * ldx;
    for (int c = off + warp; c < off + w; c += 8) {
        const __half* ar = A + (size_t)c * K;
        float acc = 0.f;
        for (int k = 2 * lane; k < K; k += 64) {
            const float2 av = __half22float2(*reinterpret_cast<const __half2*>(ar + k));
            float2 xv;
            if (x_hi) {
                const float2 h = __half22float2(*reinterpret_cast<const __half2*>(x_hi + xr + k));
                const float2 l = __half22float2(*reinterpret_cast<const __half2*>(x_lo + xr + k));
                xv = make_float2(h.x + l.x, h.y + l.y);
            } else {
                xv = *reinterpret_cast<const float2*>(x_f32 + xr + k);
            }
            acc = fmaf(av.x, xv.x, acc);
            acc = fmaf(av.y, xv.y, acc);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) {
            const float t = s * acc;
            const __half h = __float2half_rn(t);
            t_hi[row + c] = h;
            t_lo[row + c] = __float2half_rn(t - __half2float(h));
            if (t_f32) t_f32[row + c] = t;
        }
    }
}

inline void lora_shrink(cudaStream_t st, int rows, const __half* x_hi, const __half* x_lo, const float* x_f32, int ldx, int K, const __half* A, int Rp,
                        const LoraTab* tab, int g, const int* ad, const int* act, __half* t_hi, __half* t_lo, float* t_f32) {
    AHA_REQUIRE(K % 64 == 0 && ldx % 2 == 0, "lora_shrink: K must be a multiple of 64");
    lora_shrink_kernel<<<rows, 256, 0, st>>>(x_hi, x_lo, x_f32, ldx, K, A, Rp, tab, g, ad, act, t_hi, t_lo, t_f32);
    AHA_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------------- host: the loaded adapters
struct LoraAdapter {
    uint32_t id = 0;
    int r = 0;
    float scale = 0.f;
    int w[kLoraGroups] = {0, 0, 0, 0};
    // per layer and group: A block [w][K] and B block [N][w], fp16 (empty when the group has no target in the adapter)
    std::vector<std::vector<__half>> A[kLoraGroups], B[kLoraGroups];
};

// Every adapter of a handle, and the pools and buffers the kernels read.  The pools are rebuilt whenever an adapter is created or
// destroyed; `version` counts the rebuilds (a captured step graph reads the pools' addresses and is dropped on a new version).
struct LoraSet {
    int L = 0, N[kLoraGroups] = {0, 0, 0, 0}, K[kLoraGroups] = {0, 0, 0, 0};
    std::vector<LoraAdapter> ads;             // dense index = the adapter's index in the device table
    int Rp[kLoraGroups] = {0, 0, 0, 0};
    int Rmax = 0;                             // max_g Rp[g]
    std::vector<__half*> A[kLoraGroups], B[kLoraGroups];   // [L] device pools
    LoraTab* d_tab = nullptr;
    uint64_t version = 0;
    // prefill: t of up to `pf_rows` rows, the per-row adapter index and the tail lists of the running prefill
    __half *pf_hi = nullptr, *pf_lo = nullptr;
    float* pf_f32 = nullptr;
    int* pf_ad = nullptr;
    int* pf_list = nullptr;
    size_t pf_rows = 0, pf_cols = 0;
    bool pf_on = false;                       // the running TextModel::prefill adds the tails
    std::vector<void*> mem;                   // every cudaMalloc above (pools, table, prefill buffers)

    bool any() const { return !ads.empty(); }
    int index_of(uint32_t id) const {
        for (size_t i = 0; i < ads.size(); ++i) if (ads[i].id == id) return (int)i;
        return -1;
    }
    template <typename T>
    T* dalloc(size_t n) {
        void* p = nullptr;
        AHA_CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
        mem.push_back(p);
        return reinterpret_cast<T*>(p);
    }
    void free_all() {
        for (void* p : mem) cudaFree(p);
        mem.clear();
        for (int g = 0; g < kLoraGroups; ++g) { A[g].clear(); B[g].clear(); Rp[g] = 0; }
        Rmax = 0; d_tab = nullptr; pf_hi = pf_lo = nullptr; pf_f32 = nullptr; pf_ad = pf_list = nullptr; pf_rows = pf_cols = 0;
    }
    // the pools of the adapters in `ads` (none: nothing allocated)
    void rebuild(cudaStream_t st) {
        AHA_CUDA_CHECK(cudaStreamSynchronize(st));
        free_all();
        ++version;
        if (ads.empty()) return;
        std::vector<LoraTab> tab(ads.size());
        for (int g = 0; g < kLoraGroups; ++g) {
            int off = 0;
            for (size_t i = 0; i < ads.size(); ++i) { tab[i].off[g] = off; tab[i].w[g] = ads[i].w[g]; off += ads[i].w[g]; }
            Rp[g] = ceil_div(off, kLoraKb) * kLoraKb;
            Rmax = std::max(Rmax, Rp[g]);
        }
        for (size_t i = 0; i < ads.size(); ++i) tab[i].scale = ads[i].scale;
        d_tab = dalloc<LoraTab>(tab.size());
        AHA_CUDA_CHECK(cudaMemcpy(d_tab, tab.data(), tab.size() * sizeof(LoraTab), cudaMemcpyHostToDevice));
        for (int g = 0; g < kLoraGroups; ++g) {
            A[g].assign(L, nullptr); B[g].assign(L, nullptr);
            const int R = Rp[g];
            if (R == 0) continue;
            const size_t Kg = K[g], Ng = N[g];
            std::vector<__half> a(R * Kg), b(Ng * R);
            for (int l = 0; l < L; ++l) {
                std::fill(a.begin(), a.end(), __float2half_rn(0.f));
                std::fill(b.begin(), b.end(), __float2half_rn(0.f));
                for (size_t i = 0; i < ads.size(); ++i) {
                    const LoraAdapter& ad = ads[i];
                    const int w = ad.w[g], off = tab[i].off[g];
                    if (w == 0 || ad.A[g][l].empty()) continue;
                    std::memcpy(a.data() + (size_t)off * Kg, ad.A[g][l].data(), (size_t)w * Kg * sizeof(__half));
                    for (size_t n = 0; n < Ng; ++n) std::memcpy(b.data() + n * R + off, ad.B[g][l].data() + n * w, (size_t)w * sizeof(__half));
                }
                A[g][l] = dalloc<__half>(a.size());
                B[g][l] = dalloc<__half>(b.size());
                AHA_CUDA_CHECK(cudaMemcpy(A[g][l], a.data(), a.size() * sizeof(__half), cudaMemcpyHostToDevice));
                AHA_CUDA_CHECK(cudaMemcpy(B[g][l], b.data(), b.size() * sizeof(__half), cudaMemcpyHostToDevice));
            }
        }
        pf_list = dalloc<int>((size_t)kLoraGroups * (1 + Rmax / kLoraKb));
    }
    // The tail lists of the adapters `used` (indices, any order, < 0 ignored): per group [count, k-blocks holding their columns ascending],
    // into host rows of 1 + Rmax / 64 ints.
    std::vector<int> lists(const std::vector<int>& used) const {
        const int stride = 1 + Rmax / kLoraKb;
        std::vector<int> h((size_t)kLoraGroups * stride, 0);
        for (int g = 0; g < kLoraGroups; ++g) {
            std::vector<char> on((size_t)std::max(1, Rp[g] / kLoraKb), 0);
            for (int a : used) {
                if (a < 0) continue;
                int off = 0;
                for (int i = 0; i < a; ++i) off += ads[i].w[g];
                for (int c = off; c < off + ads[a].w[g]; c += kLoraAlign) on[c / kLoraKb] = 1;
            }
            int* row = h.data() + (size_t)g * stride;
            for (int kb = 0; kb < Rp[g] / kLoraKb; ++kb) if (on[kb]) row[1 + row[0]++] = kb;
        }
        return h;
    }
    int list_stride() const { return 1 + Rmax / kLoraKb; }
    // prefill rows [0, rows) run the adapters ad[row] (indices, < 0: none): the row array and the tail lists to the device
    void prefill_begin(cudaStream_t st, const std::vector<int>& ad) {
        AHA_REQUIRE(any(), "LoRA prefill without adapters");
        const size_t rows = ad.size();
        if (rows > pf_rows || (size_t)Rmax > pf_cols) {
            AHA_CUDA_CHECK(cudaStreamSynchronize(st));
            const size_t R = std::max(rows, pf_rows), C = std::max((size_t)Rmax, pf_cols);
            pf_hi = dalloc<__half>(R * C); pf_lo = dalloc<__half>(R * C); pf_f32 = dalloc<float>(R * C); pf_ad = dalloc<int>(R);
            pf_rows = R; pf_cols = C;
        }
        std::vector<int> used(ad);
        std::sort(used.begin(), used.end());
        used.erase(std::unique(used.begin(), used.end()), used.end());
        const std::vector<int> h = lists(used);
        AHA_CUDA_CHECK(cudaMemcpyAsync(pf_ad, ad.data(), rows * sizeof(int), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaMemcpyAsync(pf_list, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        AHA_CUDA_CHECK(cudaStreamSynchronize(st));   // host vectors
        pf_on = true;
    }
    void prefill_end() { pf_on = false; }
};

}  // namespace aha
