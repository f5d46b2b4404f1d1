// kernels_common.cuh -- elementwise / normalisation / gather kernels shared by text, vision and audio paths.
// All activations are fp32; linear weights are fp16 (lossless for the fp16 checkpoints) and every
// product is formed in fp32 -- the same arithmetic as the reference's Candle F32 CPU path.
#pragma once
#include "common.cuh"

namespace aha {

// Embedding::forward (row gather), fp16 table -> fp32 rows.  src/models/qwen3/model.rs:191-193
__device__ __forceinline__ void embed_row_dev(uint32_t id, const __half* __restrict__ table, float* __restrict__ out, int H, int V) {
    if (id >= (uint32_t)V) id = V - 1;  // host validates; keep the kernel memory-safe regardless
    const __half* row = table + (size_t)id * H;
    for (int i = threadIdx.x * 2; i < H; i += blockDim.x * 2) {
        float2 v = __half22float2(*reinterpret_cast<const __half2*>(row + i));
        *reinterpret_cast<float2*>(out + i) = v;
    }
}
__global__ void embed_gather_kernel(const uint32_t* __restrict__ ids, const __half* __restrict__ table,
                                    float* __restrict__ out, int S, int H, int V) {
    const int s = blockIdx.x;
    embed_row_dev(ids[s], table, out + (size_t)s * H, H, V);
}

// candle_nn RmsNorm over the last dim: x / sqrt(mean(x^2) + eps) * w.  One block per row.
__global__ void rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, float eps,
                               float* __restrict__ out, int H) {
    __shared__ float red[32];
    const float* xr = x + (size_t)blockIdx.x * H;
    float ss = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) { float v = xr[i]; ss = fmaf(v, v, ss); }
    ss = block_sum(ss, red);
    const float inv = 1.0f / sqrtf(ss / (float)H + eps);
    for (int i = threadIdx.x; i < H; i += blockDim.x) out[(size_t)blockIdx.x * H + i] = xr[i] * inv * w[i];
}

// x = hi + lo with both halves fp16 (|lo| <= 2^-11 |hi|): the operand format of the tensor-core GEMMs (gemm_tc.cuh).  Producers that feed
// a GEMM write the two halves directly instead of an fp32 tensor that a separate pass would have to read back and split.
__device__ __forceinline__ void split_half(float x, __half& h, __half& l) {
    h = __float2half_rn(x);
    l = __float2half_rn(x - __half2float(h));
}
// rmsnorm_kernel with the split output: out_hi / out_lo [rows, H] fp16.  rows != nullptr gathers: output row r is input row rows[r].
__global__ void rmsnorm_split_kernel(const float* __restrict__ x, const float* __restrict__ w, float eps, __half* __restrict__ out_hi,
                                     __half* __restrict__ out_lo, int H, const int* __restrict__ rows = nullptr) {
    __shared__ float red[32];
    const float* xr = x + (size_t)(rows ? rows[blockIdx.x] : (int)blockIdx.x) * H;
    float ss = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) { float v = xr[i]; ss = fmaf(v, v, ss); }
    ss = block_sum(ss, red);
    const float inv = 1.0f / sqrtf(ss / (float)H + eps);
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        __half h, l;
        split_half(xr[i] * inv * w[i], h, l);
        out_hi[(size_t)blockIdx.x * H + i] = h;
        out_lo[(size_t)blockIdx.x * H + i] = l;
    }
}
// layernorm_kernel with the split output
__global__ void layernorm_split_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b, float eps,
                                       __half* __restrict__ out_hi, __half* __restrict__ out_lo, int H) {
    __shared__ float red[32];
    const float* xr = x + (size_t)blockIdx.x * H;
    float s = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) s += xr[i];
    const float mean = block_sum(s, red) / (float)H;
    float v = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) { float d = xr[i] - mean; v = fmaf(d, d, v); }
    const float inv = 1.0f / sqrtf(block_sum(v, red) / (float)H + eps);
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        __half h, l;
        split_half((xr[i] - mean) * inv * w[i] + b[i], h, l);
        out_hi[(size_t)blockIdx.x * H + i] = h;
        out_lo[(size_t)blockIdx.x * H + i] = l;
    }
}

// candle_nn LayerNorm (remove_mean, affine): (x-mean)/sqrt(var+eps)*w+b.  One block per row of length H.
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                 const float* __restrict__ b, float eps, float* __restrict__ out, int H) {
    __shared__ float red[32];
    const float* xr = x + (size_t)blockIdx.x * H;
    float s = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) s += xr[i];
    const float mean = block_sum(s, red) / (float)H;
    float v = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) { float d = xr[i] - mean; v = fmaf(d, d, v); }
    const float inv = 1.0f / sqrtf(block_sum(v, red) / (float)H + eps);
    for (int i = threadIdx.x; i < H; i += blockDim.x)
        out[(size_t)blockIdx.x * H + i] = (xr[i] - mean) * inv * w[i] + b[i];
}

// out[idx[r], :] = src[r, :]   (masked_scatter_dim0, src/utils/tensor_utils.rs:294-321)
// add != 0: out[idx[r], :] += src[r, :]   (mask_index_add, tensor_utils.rs:466-470)
__global__ void scatter_rows_kernel(const int* __restrict__ idx, const float* __restrict__ src,
                                    float* __restrict__ out, int H, int add) {
    const int r = blockIdx.x;
    float* o = out + (size_t)idx[r] * H;
    const float* s = src + (size_t)r * H;
    for (int i = threadIdx.x; i < H; i += blockDim.x) o[i] = add ? (o[i] + s[i]) : s[i];
}

// out[r] = src[idx[r]] (rows of H floats), one block per output row
__global__ void gather_rows_kernel(const int* __restrict__ idx, const float* __restrict__ src, float* __restrict__ out, int H) {
    const int r = blockIdx.x;
    const float* s = src + (size_t)idx[r] * H;
    float* o = out + (size_t)r * H;
    for (int i = threadIdx.x; i < H; i += blockDim.x) o[i] = s[i];
}

// l2_normalize (src/models/common/modules.rs:1287-1294): x / sqrt(sum(x^2) + 1e-6), one row per block.
__global__ void l2_normalize_kernel(const float* __restrict__ x, float* __restrict__ out, int H) {
    __shared__ float red[32];
    const float* xr = x + (size_t)blockIdx.x * H;
    float ss = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) ss = fmaf(xr[i], xr[i], ss);
    ss = block_sum(ss, red);
    const float inv = 1.0f / sqrtf(ss + 1e-6f);
    for (int i = threadIdx.x; i < H; i += blockDim.x) out[(size_t)blockIdx.x * H + i] = xr[i] * inv;
}

__global__ void add_inplace_kernel(float* __restrict__ x, const float* __restrict__ y, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] += y[i];
}

// Two-stage argmax, "first maximal index" like candle's Sampling::ArgMax.
// Stage 1 is fused into the lm_head GEMV epilogue where possible; this standalone version covers logits[V].
__device__ __forceinline__ void argmax_partial_dev(const float* __restrict__ logits, int V, float* __restrict__ pmax, int* __restrict__ pidx,
                                                   float* smax, int* sidx) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < V; i += gridDim.x * blockDim.x) {
        float v = logits[i];
        if (v > best || (v == best && i < bi)) { best = v; bi = i; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) { smax[wid] = best; sidx[wid] = bi; }
    __syncthreads();
    if (wid == 0) {
        const int nw = blockDim.x >> 5;
        best = lane < nw ? smax[lane] : -INFINITY;
        bi = lane < nw ? sidx[lane] : 0x7fffffff;
        for (int o = 16; o > 0; o >>= 1) {
            float ov = __shfl_xor_sync(0xffffffffu, best, o);
            int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if (lane == 0) { pmax[blockIdx.x] = best; pidx[blockIdx.x] = bi; }
    }
}
__global__ void argmax_partial_kernel(const float* __restrict__ logits, int V, float* __restrict__ pmax,
                                      int* __restrict__ pidx) {
    __shared__ float smax[32];
    __shared__ int sidx[32];
    argmax_partial_dev(logits, V, pmax, pidx, smax, sidx);
}
// the same over nb logits rows (ld floats apart): blockIdx.y = row, gridDim.x candidates per row (pmax / pidx [nb][gridDim.x])
__global__ void argmax_partial_rows_kernel(const float* __restrict__ logits, int ld, int V, float* __restrict__ pmax, int* __restrict__ pidx) {
    __shared__ float smax[32];
    __shared__ int sidx[32];
    const size_t r = blockIdx.y;
    argmax_partial_dev(logits + r * ld, V, pmax + r * gridDim.x, pidx + r * gridDim.x, smax, sidx);
}

// Stage 2: reduce the per-block candidates, publish the token, and advance the device-side decode state:
// state[0] = next token, state[1] = position of the next token (ctx so far), history[state[2]++] = token.
struct DecodeState {
    uint32_t token;      // input token of the next step
    int32_t pos;         // seqlen_offset of the next step (= tokens already cached)
    int32_t rope_delta;  // Qwen3-VL rope_deltas (0 for text / ASR)
    int32_t n_hist;      // tokens written to history
    uint32_t n_draws;    // random draws the request's sampler has consumed (index into its ChaCha12 stream)
    uint32_t fsm_state;  // state of the request's token automaton (sampling.cuh; 0 and unused without one)
    uint32_t pad_[2];
};
__device__ __forceinline__ void argmax_final_dev(const float* __restrict__ pmax, const int* __restrict__ pidx, int n,
                                                 uint32_t* __restrict__ argmax_out, DecodeState* __restrict__ st,
                                                 uint32_t* __restrict__ history, int hist_cap, int advance) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < n; i += 32) {
        float v = pmax[i];
        int id = pidx[i];
        if (v > best || (v == best && id < bi)) { best = v; bi = id; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (threadIdx.x == 0) {
        if (bi == 0x7fffffff) bi = 0;   // every candidate NaN: publish a valid id
        if (argmax_out) *argmax_out = (uint32_t)bi;
        if (advance && st) {
            st->token = (uint32_t)bi;
            st->pos += 1;
            if (history && st->n_hist < hist_cap) history[st->n_hist] = (uint32_t)bi;
            st->n_hist += 1;
        }
    }
}
__global__ void argmax_final_kernel(const float* __restrict__ pmax, const int* __restrict__ pidx, int n,
                                    uint32_t* __restrict__ argmax_out, DecodeState* __restrict__ st,
                                    uint32_t* __restrict__ history, int hist_cap, int advance) {
    argmax_final_dev(pmax, pidx, n, argmax_out, st, history, hist_cap, advance);
}

// Row-indexed kernels of a wide batch step (batch_decode.cuh): row j belongs to slot act[j], read from device memory so that one launch
// (and one captured graph) serves every composition of the same width.
__global__ void embed_rows_kernel(const int* __restrict__ act, const DecodeState* __restrict__ st, const __half* __restrict__ table,
                                  float* __restrict__ out, int H, int V) {
    embed_row_dev(st[act[blockIdx.x]].token, table, out + (size_t)blockIdx.x * H, H, V);
}
// stage 2 of row j (one warp per row): the slot's token, decode state and history
__global__ void argmax_final_rows_kernel(const float* __restrict__ pmax, const int* __restrict__ pidx, int n, const int* __restrict__ act,
                                         uint32_t* __restrict__ tok, DecodeState* __restrict__ st, uint32_t* __restrict__ hist, int hist_cap,
                                         int advance) {
    const int j = blockIdx.x, slot = act[j];
    argmax_final_dev(pmax + (size_t)j * n, pidx + (size_t)j * n, n, tok + slot, st + slot, hist + (size_t)slot * hist_cap, hist_cap, advance);
}

}  // namespace aha
