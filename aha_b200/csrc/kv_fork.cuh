// kv_fork.cuh -- OpenAI `n` (aha_b200_batch_add_n): the prompt's K/V pages of one batch slot copied into the pages of other slots.
//
// One page of one layer is a contiguous run of page_stride = 2 * nkv * kPage * hd fp32 values (the K block, then the V block, text_model.cuh
// kv_src), so the copy moves whole pages and never looks inside one.  A CTA owns 1 / split of one (layer, logical page): it reads the source
// slot's physical page from its table row, loads each 16-byte vector of its part once (streaming load) and stores it to the same logical page
// of every destination.  Bytes moved: P read + (n_dst) * P written, P = layers * pages * page_stride * 4.
#pragma once
#include <algorithm>

#include "text_model.cuh"

namespace aha {

constexpr int kForkMaxDst = 63;          // a wide session holds 64 slots: one source, at most 63 destinations
constexpr int kForkThreads = 256;
constexpr int kForkUnroll = 4;           // vectors in flight per thread before the stores

struct KvForkArgs {
    float* pool;                         // TextModel::kv_pool
    size_t layer_stride, page_stride;    // floats
    const int* tables;                   // [rows][num_pages] device page tables (BatchDecoder::d_tables)
    int num_pages;
    int src, n_dst;                      // table rows
    int dst[kForkMaxDst];
    int split;                           // CTAs per (layer, page)
};

__global__ void __launch_bounds__(kForkThreads) kv_fork_kernel(const KvForkArgs a) {
    __shared__ int dpage[kForkMaxDst];
    const int p = blockIdx.x / a.split, part = blockIdx.x % a.split;
    for (int j = threadIdx.x; j < a.n_dst; j += kForkThreads) dpage[j] = a.tables[(size_t)a.dst[j] * a.num_pages + p];
    __syncthreads();
    float* layer = a.pool + (size_t)blockIdx.y * a.layer_stride;
    const float4* src = reinterpret_cast<const float4*>(layer + (size_t)a.tables[(size_t)a.src * a.num_pages + p] * a.page_stride);
    const size_t n4 = a.page_stride / 4, per = (n4 + a.split - 1) / a.split;
    const size_t b = (size_t)part * per, e = min(n4, b + per);
    for (size_t i = b + threadIdx.x; i < e; i += (size_t)kForkThreads * kForkUnroll) {
        float4 v[kForkUnroll];
#pragma unroll
        for (int u = 0; u < kForkUnroll; ++u) {
            const size_t k = i + (size_t)u * kForkThreads;
            if (k < e) v[u] = __ldcs(src + k);
        }
        for (int j = 0; j < a.n_dst; ++j) {
            float4* dst = reinterpret_cast<float4*>(layer + (size_t)dpage[j] * a.page_stride);
#pragma unroll
            for (int u = 0; u < kForkUnroll; ++u) {
                const size_t k = i + (size_t)u * kForkThreads;
                if (k < e) dst[k] = v[u];
            }
        }
    }
}

// logical pages 0 .. pages-1 of table row src, every layer, into the same logical pages of rows dst (one launch).  Every destination row
// must already map those pages.  The split gives the grid about four CTAs per SM, but never less than one unrolled pass per CTA.
inline void kv_fork(Ctx& c, float* pool, size_t layer_stride, size_t page_stride, int layers, const int* tables, int num_pages, int src,
                    const int* dst, int n_dst, int pages) {
    AHA_REQUIRE(n_dst >= 1 && n_dst <= kForkMaxDst, "kv_fork: 1 to 63 destinations");
    AHA_REQUIRE(pages >= 1 && pages <= num_pages && page_stride % 4 == 0, "kv_fork: bad page range");
    KvForkArgs a{};
    a.pool = pool; a.layer_stride = layer_stride; a.page_stride = page_stride; a.tables = tables; a.num_pages = num_pages;
    a.src = src; a.n_dst = n_dst;
    for (int j = 0; j < n_dst; ++j) a.dst[j] = dst[j];
    const int max_split = std::max<int>(1, (int)(page_stride / 4 / (kForkThreads * kForkUnroll)));
    a.split = std::min(max_split, std::max(1, ceil_div(4 * c.num_sms, layers * pages)));
    kv_fork_kernel<<<dim3((unsigned)(pages * a.split), (unsigned)layers), kForkThreads, 0, c.stream>>>(a);
    c.cnt.kernels++;
    AHA_CUDA_CHECK(cudaGetLastError());
}

}  // namespace aha
