// vb_heads.cu — fused softmax cross-entropy over bf16 logits for the masked-LM head
// (reference modeling.py:1471-1473: CrossEntropyLoss(ignore_index=-1) on prediction_scores; SURVEY.md §8f rank 1).
//
// HBM-bound row kernels: one CTA per labelled row, the row (vocab ~30.5 k bf16 = 61 KB) is streamed with 16-byte
// loads. Forward: online log-sum-exp -> lse[row], loss[row] = lse - logit[label]. Backward: the gradient
// (softmax - onehot) * scale overwrites the logits in place (they are not needed afterwards), in bf16 — the
// operand the decoder's dgrad / wgrad GEMMs consume. PyTorch's path (fp32 copy + log_softmax + nll + 2 backward
// passes) moved ~6x the bytes.
#include "vb_internal.h"

namespace vb {

constexpr int kCeThreads = 256;

__device__ __forceinline__ float block_max(float v, float* sh) {
    v = warp_max(v);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = sh[0];
#pragma unroll
    for (int i = 1; i < kCeThreads / 32; ++i) r = fmaxf(r, sh[i]);
    __syncthreads();
    return r;
}
__device__ __forceinline__ float block_sum(float v, float* sh) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = 0.f;
#pragma unroll
    for (int i = 0; i < kCeThreads / 32; ++i) r += sh[i];
    __syncthreads();
    return r;
}

// logits [rows, ld] bf16, valid columns [0, vocab); labels int64 [rows] in [0, vocab)
__global__ void __launch_bounds__(kCeThreads)
ce_fwd_kernel(const bf16* __restrict__ logits, long long ld, const long long* __restrict__ labels, int vocab,
              float* __restrict__ lse_out, float* __restrict__ loss_out) {
    __shared__ float sh[kCeThreads / 32];
    const long long row = blockIdx.x;
    const bf16* x = logits + row * ld;
    const int chunks = vocab >> 3;
    float m = -INFINITY, s = 0.f;  // per-thread online max / sum of exp2((x - m) * log2e)
    for (int ch = threadIdx.x; ch < chunks; ch += kCeThreads) {
        const uint4 u = ldg_v4(x + ch * 8);
        const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
        const float v[8] = {a.x, a.y, b.x, b.y, c.x, c.y, d.x, d.y};
        float cm = v[0];
#pragma unroll
        for (int i = 1; i < 8; ++i) cm = fmaxf(cm, v[i]);
        const float nm = fmaxf(m, cm);
        float acc = s * fast_ex2((m - nm) * 1.4426950408889634f);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc += fast_ex2((v[i] - nm) * 1.4426950408889634f);
        s = acc;
        m = nm;
    }
    for (int col = (chunks << 3) + threadIdx.x; col < vocab; col += kCeThreads) {  // tail (vocab % 8)
        const float v = __bfloat162float(x[col]);
        const float nm = fmaxf(m, v);
        s = s * fast_ex2((m - nm) * 1.4426950408889634f) + fast_ex2((v - nm) * 1.4426950408889634f);
        m = nm;
    }
    const float gm = block_max(m, sh);
    const float gs = block_sum(m == -INFINITY ? 0.f : s * fast_ex2((m - gm) * 1.4426950408889634f), sh);
    if (threadIdx.x == 0) {
        const float lse = gm + logf(gs);
        lse_out[row] = lse;
        // a label outside [0, vocab) (e.g. an ignore index) contributes no loss and, in ce_bwd_kernel, no gradient:
        // never an out-of-bounds read
        const long long lab = labels[row];
        loss_out[row] = (lab >= 0 && lab < vocab) ? lse - __bfloat162float(x[lab]) : 0.f;
    }
}

// logits <- (softmax(logits) - onehot(label)) * scale, columns >= vocab (padding up to ld_valid) <- 0
__global__ void __launch_bounds__(kCeThreads)
ce_bwd_kernel(bf16* __restrict__ logits, long long ld, const long long* __restrict__ labels, int vocab, int padded,
              const float* __restrict__ lse, const float* __restrict__ scale_ptr) {
    const long long row = blockIdx.x;
    bf16* x = logits + row * ld;
    const float l2 = lse[row] * 1.4426950408889634f;
    const float scale = *scale_ptr;
    const long long lab = labels[row];
    const bool ignored = lab < 0 || lab >= vocab;
    const int label = ignored ? -1 : static_cast<int>(lab);
    const int chunks = padded >> 3;
    for (int ch = threadIdx.x; ch < chunks; ch += kCeThreads) {
        const uint4 u = *reinterpret_cast<const uint4*>(x + ch * 8);
        const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
        float v[8] = {a.x, a.y, b.x, b.y, c.x, c.y, d.x, d.y};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int col = ch * 8 + i;
            float g = (col < vocab && !ignored) ? fast_ex2(fmaf(v[i], 1.4426950408889634f, -l2)) : 0.f;
            if (col == label) g -= 1.f;
            v[i] = g * scale;
        }
        uint4 o;
        o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
        o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
        *reinterpret_cast<uint4*>(x + ch * 8) = o;
    }
}

int ce_fwd(const void* logits, long long ld, const long long* labels, int rows, int vocab, float* lse, float* loss,
           cudaStream_t st) {
    VB_REQUIRE(rows >= 0 && vocab > 0 && ld >= vocab && ld % 8 == 0, "cross-entropy: bad shape rows=%d vocab=%d ld=%lld", rows, vocab, ld);
    VB_REQUIRE(all_aligned16(logits), "cross-entropy: logits must be 16-byte aligned");
    if (rows == 0) return 0;
    {
        ProfScope ps(st, PROF_OTHER, 2.0 * rows * vocab, 1);
        ce_fwd_kernel<<<rows, kCeThreads, 0, st>>>(static_cast<const bf16*>(logits), ld, labels, vocab, lse, loss);
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int ce_bwd(void* logits, long long ld, const long long* labels, int rows, int vocab, int padded, const float* lse,
           const float* scale, cudaStream_t st) {
    VB_REQUIRE(rows >= 0 && vocab > 0 && padded >= vocab && padded % 8 == 0 && ld >= padded && ld % 8 == 0,
               "cross-entropy backward: bad shape");
    VB_REQUIRE(all_aligned16(logits), "cross-entropy backward: logits must be 16-byte aligned");
    if (rows == 0) return 0;
    {
        ProfScope ps(st, PROF_OTHER, 4.0 * rows * padded, 1);
        ce_bwd_kernel<<<rows, kCeThreads, 0, st>>>(static_cast<bf16*>(logits), ld, labels, vocab, padded, lse, scale);
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace vb

extern "C" {
int vb_cross_entropy_fwd(const void* logits, int64_t ld, const int64_t* labels, int32_t rows, int32_t vocab, float* lse,
                         float* loss_rows, void* stream) {
    return vb::ce_fwd(logits, ld, reinterpret_cast<const long long*>(labels), rows, vocab, lse, loss_rows,
                      static_cast<cudaStream_t>(stream));
}
int vb_cross_entropy_bwd(void* logits, int64_t ld, const int64_t* labels, int32_t rows, int32_t vocab, int32_t padded_cols,
                         const float* lse, const float* scale, void* stream) {
    return vb::ce_bwd(logits, ld, reinterpret_cast<const long long*>(labels), rows, vocab, padded_cols, lse, scale,
                      static_cast<cudaStream_t>(stream));
}
}
