// vb_optim.cu — multi-tensor BertAdam step (SURVEY.md §8f rank 2).
// Reference: visualbert/pytorch_pretrained_bert/optimization.py:239-304 — a Python loop over ~200 parameter tensors,
// ~10 elementwise launches each plus a per-parameter clip_grad_norm_. Here the whole step is two launches over a
// device table of tensors:
//   1. adam_sumsq_kernel   sum of squares of every gradient tensor (for the PER-PARAMETER clip, opt.py:272-273)
//   2. adam_update_kernel  g' = g * min(1, max_norm / (||g|| + 1e-6)); m = b1 m + (1-b1) g'; v = b2 v + (1-b2) g'^2;
//                          p -= lr * (m / (sqrt(v) + eps) + wd * p)        (no bias correction, decoupled decay)
// Both are HBM-bound: 4 B/param for (1), 28 B/param for (2) (read p, g, m, v; write p, m, v) — 32 B/param per step.
// Work is cut in chunks of VB_ADAM_CHUNK elements; one CTA per chunk finds its tensor by binary search in the table.
#include "vb_internal.h"

namespace vb {

constexpr int kAdamThreads = 256;
constexpr int kAdamChunk = VB_ADAM_CHUNK;

__device__ __forceinline__ int find_tensor(const vb_adam_tensor* __restrict__ tab, int n, int chunk) {
    int lo = 0, hi = n - 1;  // last entry with first_chunk <= chunk
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tab[mid].first_chunk <= chunk) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// PART = false: the chunk's sum of squares is atomically added to sumsq[tensor]. PART = true (deterministic mode): it is stored
// to sumsq[chunk] (the workspace), and adam_update_ordered_kernel adds a tensor's chunk sums in chunk order.
template <bool PART>
__device__ __forceinline__ void adam_sumsq_body(const vb_adam_tensor* __restrict__ tab, int n_tensors, float* __restrict__ sumsq) {
    __shared__ float sh[kAdamThreads / 32];
    const int t = find_tensor(tab, n_tensors, blockIdx.x);
    const vb_adam_tensor e = tab[t];
    const long long begin = static_cast<long long>(blockIdx.x - e.first_chunk) * kAdamChunk;
    const long long end = min(begin + kAdamChunk, static_cast<long long>(e.numel));
    const float* g = static_cast<const float*>(e.g);
    float s = 0.f;
    if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
        const long long v4_end = begin + ((end - begin) & ~3LL);
        for (long long i = begin + threadIdx.x * 4LL; i < v4_end; i += kAdamThreads * 4LL) {
            const float4 x = *reinterpret_cast<const float4*>(g + i);
            s += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
        }
        for (long long i = v4_end + threadIdx.x; i < end; i += kAdamThreads) s += g[i] * g[i];
    } else {
        for (long long i = begin + threadIdx.x; i < end; i += kAdamThreads) s += g[i] * g[i];
    }
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float r = 0.f;
#pragma unroll
        for (int i = 0; i < kAdamThreads / 32; ++i) r += sh[i];
        if constexpr (PART) sumsq[blockIdx.x] = r;
        else atomicAdd(sumsq + t, r);
    }
}
__global__ void __launch_bounds__(kAdamThreads)
adam_sumsq_kernel(const vb_adam_tensor* __restrict__ tab, int n_tensors, float* __restrict__ sumsq) { adam_sumsq_body<false>(tab, n_tensors, sumsq); }
__global__ void __launch_bounds__(kAdamThreads)
adam_sumsq_part_kernel(const vb_adam_tensor* __restrict__ tab, int n_tensors, float* __restrict__ part) { adam_sumsq_body<true>(tab, n_tensors, part); }

struct AdamHyper { float b1, one_minus_b1, b2, one_minus_b2, eps, max_grad_norm; };

__device__ __forceinline__ void adam_elem(float& p, float g, float& m, float& v, float coef, float lr, float wd,
                                          const AdamHyper& h) {
    g *= coef;
    m = m * h.b1 + h.one_minus_b1 * g;
    v = v * h.b2 + h.one_minus_b2 * g * g;
    float upd = __fdiv_rn(m, __fsqrt_rn(v) + h.eps);
    if (wd > 0.f) upd += wd * p;
    p -= lr * upd;
}

// ORDERED = false: sumsq[t] is the tensor's sum of squares. ORDERED = true: sumsq holds one partial per chunk, and every CTA of
// the tensor sums them in the same fixed order (thread i takes chunks i, i + 256, ... in order, then a fixed reduction tree).
template <bool ORDERED>
__device__ __forceinline__ void adam_update_body(const vb_adam_tensor* __restrict__ tab, int n_tensors, const float* __restrict__ sumsq,
                                                 const AdamHyper& h) {
    const int t = find_tensor(tab, n_tensors, blockIdx.x);
    const vb_adam_tensor e = tab[t];
    const long long begin = static_cast<long long>(blockIdx.x - e.first_chunk) * kAdamChunk;
    const long long end = min(begin + kAdamChunk, static_cast<long long>(e.numel));
    float coef = 1.f;
    if (h.max_grad_norm > 0.f) {  // torch.nn.utils.clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), applied if < 1
        float ss;
        if constexpr (ORDERED) {
            __shared__ float sh[kAdamThreads / 32];
            const int nch = static_cast<int>((e.numel + kAdamChunk - 1) / kAdamChunk);
            float s = 0.f;
            for (int i = threadIdx.x; i < nch; i += kAdamThreads) s += sumsq[e.first_chunk + i];
            s = warp_sum(s);
            if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
            __syncthreads();
            ss = 0.f;
#pragma unroll
            for (int i = 0; i < kAdamThreads / 32; ++i) ss += sh[i];
        } else {
            ss = sumsq[t];
        }
        const float c = h.max_grad_norm / (sqrtf(ss) + 1e-6f);
        coef = c < 1.f ? c : 1.f;
    }
    float* p = static_cast<float*>(e.p);
    const float* g = static_cast<const float*>(e.g);
    float* m = static_cast<float*>(e.m);
    float* v = static_cast<float*>(e.v);
    const float lr = e.lr, wd = e.weight_decay;
    const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                           reinterpret_cast<uintptr_t>(v)) & 15) == 0;
    long long scalar_from = begin;
    if (aligned) {
        const long long v4_end = begin + ((end - begin) & ~3LL);
        for (long long i = begin + threadIdx.x * 4LL; i < v4_end; i += kAdamThreads * 4LL) {
            float4 pp = *reinterpret_cast<const float4*>(p + i);
            const float4 gg = *reinterpret_cast<const float4*>(g + i);
            float4 mm = *reinterpret_cast<const float4*>(m + i);
            float4 vv = *reinterpret_cast<const float4*>(v + i);
            adam_elem(pp.x, gg.x, mm.x, vv.x, coef, lr, wd, h);
            adam_elem(pp.y, gg.y, mm.y, vv.y, coef, lr, wd, h);
            adam_elem(pp.z, gg.z, mm.z, vv.z, coef, lr, wd, h);
            adam_elem(pp.w, gg.w, mm.w, vv.w, coef, lr, wd, h);
            *reinterpret_cast<float4*>(p + i) = pp;
            *reinterpret_cast<float4*>(m + i) = mm;
            *reinterpret_cast<float4*>(v + i) = vv;
        }
        scalar_from = v4_end;
    }
    for (long long i = scalar_from + threadIdx.x; i < end; i += kAdamThreads) {
        float pp = p[i], mm = m[i], vv = v[i];
        adam_elem(pp, g[i], mm, vv, coef, lr, wd, h);
        p[i] = pp; m[i] = mm; v[i] = vv;
    }
}
__global__ void __launch_bounds__(kAdamThreads)
adam_update_kernel(const vb_adam_tensor* __restrict__ tab, int n_tensors, const float* __restrict__ sumsq, const AdamHyper h) {
    adam_update_body<false>(tab, n_tensors, sumsq, h);
}
__global__ void __launch_bounds__(kAdamThreads)
adam_update_ordered_kernel(const vb_adam_tensor* __restrict__ tab, int n_tensors, const float* __restrict__ part, const AdamHyper h) {
    adam_update_body<true>(tab, n_tensors, part, h);
}

int bert_adam_step(const vb_adam_tensor* table, int n_tensors, int n_chunks, float* sumsq, double b1, double b2, double eps,
                   double max_grad_norm, cudaStream_t st) {
    VB_REQUIRE(table != nullptr && sumsq != nullptr, "vb_bert_adam_step: null table / scratch");
    VB_REQUIRE(n_tensors > 0 && n_chunks >= n_tensors, "vb_bert_adam_step: bad tensor / chunk counts");
    VB_REQUIRE(b1 >= 0.0 && b1 < 1.0 && b2 >= 0.0 && b2 < 1.0 && eps >= 0.0, "vb_bert_adam_step: bad b1 / b2 / eps");
    // the reference holds b1 / b2 as Python doubles and forms (1 - b) in double before it meets the fp32 tensors
    const AdamHyper h{static_cast<float>(b1), static_cast<float>(1.0 - b1), static_cast<float>(b2), static_cast<float>(1.0 - b2),
                      static_cast<float>(eps), static_cast<float>(max_grad_norm)};
    const DetWs det = det_ws();
    if (det.ptr != nullptr) {
        VB_TRY_RC(det_require(4LL * n_chunks, "vb_bert_adam_step"));
        float* part = static_cast<float*>(det.ptr);
        if (max_grad_norm > 0.0) {
            ProfScope ps(st, PROF_OTHER, 0.0, 1);
            adam_sumsq_part_kernel<<<n_chunks, kAdamThreads, 0, st>>>(table, n_tensors, part);
        }
        {
            ProfScope ps(st, PROF_OTHER, 0.0, 1);
            adam_update_ordered_kernel<<<n_chunks, kAdamThreads, 0, st>>>(table, n_tensors, part, h);
        }
        VB_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    if (max_grad_norm > 0.0) {
        VB_CHECK_CUDA(cudaMemsetAsync(sumsq, 0, sizeof(float) * n_tensors, st));
        ProfScope ps(st, PROF_OTHER, 0.0, 1);
        adam_sumsq_kernel<<<n_chunks, kAdamThreads, 0, st>>>(table, n_tensors, sumsq);
    }
    {
        ProfScope ps(st, PROF_OTHER, 0.0, 1);
        adam_update_kernel<<<n_chunks, kAdamThreads, 0, st>>>(table, n_tensors, sumsq, h);
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------
// multi-tensor cast: the bf16 compute copies of ALL weight matrices (and fp32 copies of the packed qkv biases) of a
// model are refreshed by one launch over a device table — the caller does this at the start of every training-mode
// forward, so any optimizer that updates the fp32 masters (in place, through .data, fused, ...) is picked up.
// ---------------------------------------------------------------------------------------------
constexpr int kCastChunk = VB_CAST_CHUNK;
__global__ void __launch_bounds__(256)
cast_multi_kernel(const vb_cast_item* __restrict__ tab, int n_items) {
    int lo = 0, hi = n_items - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tab[mid].first_chunk <= static_cast<int>(blockIdx.x)) lo = mid; else hi = mid - 1;
    }
    const vb_cast_item e = tab[lo];
    const long long begin = static_cast<long long>(blockIdx.x - e.first_chunk) * kCastChunk;
    const long long end = min(begin + kCastChunk, static_cast<long long>(e.numel));
    const float* src = static_cast<const float*>(e.src);
    if (e.dst_fp32) {
        float* dst = static_cast<float*>(e.dst);
        for (long long i = begin + threadIdx.x; i < end; i += 256) dst[i] = src[i];
        return;
    }
    bf16* dst = static_cast<bf16*>(e.dst);
    if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) {
        const long long v8_end = begin + ((end - begin) & ~7LL);
        for (long long i = begin + threadIdx.x * 8LL; i < v8_end; i += 256 * 8LL) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(src + i));
            const float4 b = __ldg(reinterpret_cast<const float4*>(src + i + 4));
            uint4 u;
            u.x = pack_bf16x2(a.x, a.y); u.y = pack_bf16x2(a.z, a.w);
            u.z = pack_bf16x2(b.x, b.y); u.w = pack_bf16x2(b.z, b.w);
            *reinterpret_cast<uint4*>(dst + i) = u;
        }
        for (long long i = v8_end + threadIdx.x; i < end; i += 256) dst[i] = __float2bfloat16_rn(src[i]);
    } else {
        for (long long i = begin + threadIdx.x; i < end; i += 256) dst[i] = __float2bfloat16_rn(src[i]);
    }
}

int cast_multi(const vb_cast_item* table, int n_items, int n_chunks, cudaStream_t st) {
    VB_REQUIRE(table != nullptr && n_items > 0 && n_chunks > 0, "vb_cast_multi: empty table");
    {
        ProfScope ps(st, PROF_OTHER, 0.0, 1);
        cast_multi_kernel<<<n_chunks, 256, 0, st>>>(table, n_items);
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace vb

extern "C" {
int vb_cast_multi(const vb_cast_item* table, int32_t n_items, int32_t n_chunks, void* stream) {
    return vb::cast_multi(table, n_items, n_chunks, static_cast<cudaStream_t>(stream));
}
int vb_bert_adam_step(const vb_adam_tensor* table, int32_t n_tensors, int32_t n_chunks, float* sumsq, double b1, double b2,
                      double eps, double max_grad_norm, void* stream) {
    return vb::bert_adam_step(table, n_tensors, n_chunks, sumsq, b1, b2, eps, max_grad_norm, static_cast<cudaStream_t>(stream));
}
}
