// kv_swap.cuh -- suspend / resume of a batch-session request (aha_b200_batch_suspend / _resume): its KV pages moved between the device pool
// and a pinned host arena.
//
// The arena (aha_b200_batch_swap_space) is one cudaHostAlloc-ed block of host pages; a host page holds one KV page of every layer,
// [layer][page_stride] fp32, so it is one contiguous run of L * page_stride values.  In the pool the same page of consecutive layers lies
// layer_stride apart, so one (logical page, host page) pair is one strided copy: L rows of page_stride values, pitch layer_stride on the
// device and page_stride on the host.  The copy engine moves each page with one cudaMemcpy2DAsync on the library stream.
//
// Why the copy engine and not a kernel that reads and writes the arena in place through its mapped pointer: on one H100 80GB HBM3 (700 W,
// PCIe) such a kernel (kv_fork_kernel's structure, 16-byte vectors, four loads in flight per thread) reached 50.6 GB/s out and only
// 28.6 GB/s in for a 2048-token Qwen3-0.6B context (477 MB), against 53.0 / 48.0 GB/s for these copies (profiles/run_swap.py,
// BASELINE §4): loads from host memory issued by the SMs do not keep PCIe busy.
#pragma once
#include "text_model.cuh"

namespace aha {

// logical pages 0 .. pages-1 of a page table (host copy: logical page p -> pool page table[p]), every layer, to (out) or from (!out) the
// host pages host_pages[0 .. pages-1] of the arena at `host`
inline void kv_swap(Ctx& c, bool out, float* pool, size_t layer_stride, size_t page_stride, int layers, const int* table, const int* host_pages,
                    float* host, int pages) {
    AHA_REQUIRE(pages >= 1, "kv_swap: bad page range");
    const size_t row = page_stride * sizeof(float);
    for (int p = 0; p < pages; ++p) {
        float* dev = pool + (size_t)table[p] * page_stride;
        float* h = host + (size_t)host_pages[p] * layers * page_stride;
        if (out) AHA_CUDA_CHECK(cudaMemcpy2DAsync(h, row, dev, layer_stride * sizeof(float), row, (size_t)layers, cudaMemcpyDeviceToHost, c.stream));
        else AHA_CUDA_CHECK(cudaMemcpy2DAsync(dev, layer_stride * sizeof(float), h, row, row, (size_t)layers, cudaMemcpyHostToDevice, c.stream));
    }
}

}  // namespace aha
