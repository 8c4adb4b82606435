// vb_embed.cu — BertEmbeddingsWithVisualEmbedding (reference modeling.py:1198-1257) and the small
// HBM-bound helpers around the GEMMs.
//
//  embed_fwd   text rows  = word[ids] + pos[s] + type[token_type]            (modeling.py:1213-1217)
//              visual rows = projection(feat) + pos_vis[0] + type_vis[vtype] (modeling.py:1220-1221,1247-1250)
//              rows of one example are written text-first / visual-after straight into the layer-0 input
//              [B, T+V, H] (no torch.cat, modeling.py:1253), then the joint LayerNorm (1255) and dropout (1256),
//              all in one pass with the row held in registers.
//  embed_bwd   scatter of the pre-LayerNorm gradient into the five embedding tables (fp32 atomics; the tiny
//              tables are first reduced in shared memory) and the copy of the visual rows that feeds the
//              projection's weight-gradient GEMM.
//  mask_bias   (1 - cat(input_mask, image_mask)) * -10000                    (modeling.py:1417, 1286-1294)
//  cast / colsum / fill helpers.
#include <cub/device/device_radix_sort.cuh>

#include "vb_internal.h"

namespace vb {

constexpr int kEmbWarps = 8;

__device__ __forceinline__ int clampi(long long v, int hi) { return v < 0 ? 0 : (v >= hi ? hi - 1 : static_cast<int>(v)); }

// OFF: the dropout seed is p.drop_seed + *p.drop_offset (vb_set_dropout_offset)
template <int NC, bool OFF>
__device__ __forceinline__ void embed_fwd_body(const EmbedParams& p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int S = p.T + p.V;
    const long long row = static_cast<long long>(blockIdx.x) * kEmbWarps + warp;
    if (row >= static_cast<long long>(p.B) * S) return;
    const int b = static_cast<int>(row / S), s = static_cast<int>(row % S);
    const int H = p.H, chunks = H >> 3;
    const float *r0, *r1, *r2;
    const bf16* rv = nullptr;
    if (s < p.T) {
        r0 = p.word + static_cast<long long>(clampi(p.ids[static_cast<long long>(b) * p.T + s], p.vocab)) * H;
        r1 = p.pos + static_cast<long long>(s < p.max_pos ? s : p.max_pos - 1) * H;
        r2 = p.type + static_cast<long long>(clampi(p.tt[static_cast<long long>(b) * p.T + s], p.n_types)) * H;
    } else {
        const int v = s - p.T;
        rv = p.vis_proj + (static_cast<long long>(b) * p.V + v) * H;
        r0 = nullptr;
        r1 = p.pos_vis;  // every region uses visual position row 0 (modeling.py:1247)
        r2 = p.type_vis + static_cast<long long>(clampi(p.vt[static_cast<long long>(b) * p.V + v], p.n_types)) * H;
    }
    float v[NC][8];
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        const int ch = lane + c * 32;
        if (ch < chunks) {
            float a[8];
            if (rv != nullptr) {
                const uint4 u = ldg_v4(rv + ch * 8);
                const float2 x0 = unpack_bf16x2(u.x), x1 = unpack_bf16x2(u.y), x2 = unpack_bf16x2(u.z), x3 = unpack_bf16x2(u.w);
                a[0] = x0.x; a[1] = x0.y; a[2] = x1.x; a[3] = x1.y; a[4] = x2.x; a[5] = x2.y; a[6] = x3.x; a[7] = x3.y;
            } else {
                const float4 w0 = __ldg(reinterpret_cast<const float4*>(r0 + ch * 8));
                const float4 w1 = __ldg(reinterpret_cast<const float4*>(r0 + ch * 8 + 4));
                a[0] = w0.x; a[1] = w0.y; a[2] = w0.z; a[3] = w0.w; a[4] = w1.x; a[5] = w1.y; a[6] = w1.z; a[7] = w1.w;
            }
            const float4 p0 = __ldg(reinterpret_cast<const float4*>(r1 + ch * 8));
            const float4 p1 = __ldg(reinterpret_cast<const float4*>(r1 + ch * 8 + 4));
            const float4 t0 = __ldg(reinterpret_cast<const float4*>(r2 + ch * 8));
            const float4 t1 = __ldg(reinterpret_cast<const float4*>(r2 + ch * 8 + 4));
            a[0] += p0.x + t0.x; a[1] += p0.y + t0.y; a[2] += p0.z + t0.z; a[3] += p0.w + t0.w;
            a[4] += p1.x + t1.x; a[5] += p1.y + t1.y; a[6] += p1.z + t1.z; a[7] += p1.w + t1.w;
            // the pre-LN sum is kept in bf16 for backward; normalise exactly what is stored
            uint4 u;
            u.x = pack_bf16x2(a[0], a[1]); u.y = pack_bf16x2(a[2], a[3]);
            u.z = pack_bf16x2(a[4], a[5]); u.w = pack_bf16x2(a[6], a[7]);
            stg_v4(p.pre + row * H + ch * 8, u);
            const float2 y0 = unpack_bf16x2(u.x), y1 = unpack_bf16x2(u.y), y2 = unpack_bf16x2(u.z), y3 = unpack_bf16x2(u.w);
            v[c][0] = y0.x; v[c][1] = y0.y; v[c][2] = y1.x; v[c][3] = y1.y;
            v[c][4] = y2.x; v[c][5] = y2.y; v[c][6] = y3.x; v[c][7] = y3.y;
#pragma unroll
            for (int i = 0; i < 8; ++i) sum += v[c][i];
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[c][i] = 0.f;
        }
    }
    const float mean = warp_sum(sum) / H;
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < NC; ++c)
        if (lane + c * 32 < chunks) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { const float d = v[c][i] - mean; q += d * d; }
        }
    const float rstd = rsqrtf(warp_sum(q) / H + p.eps);
    if (lane == 0) { p.mean[row] = mean; p.rstd[row] = rstd; }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        const int ch = lane + c * 32;
        if (ch < chunks) {
            float o[8];
#pragma unroll
            for (int i = 0; i < 8; ++i)
                o[i] = __ldg(p.gamma + ch * 8 + i) * ((v[c][i] - mean) * rstd) + __ldg(p.beta + ch * 8 + i);
            if (p.drop_scale != 0.f) {
                const unsigned long long e8 = (static_cast<unsigned long long>(row) * static_cast<unsigned>(H) + ch * 8) >> 3;
                const uint32_t keep = dropout_keep8(OFF ? p.drop_seed + *p.drop_offset : p.drop_seed, p.drop_stream, e8, p.drop_thresh16);
#pragma unroll
                for (int i = 0; i < 8; ++i) o[i] = ((keep >> i) & 1u) ? o[i] * p.drop_scale : 0.f;
            }
            uint4 u;
            u.x = pack_bf16x2(o[0], o[1]); u.y = pack_bf16x2(o[2], o[3]);
            u.z = pack_bf16x2(o[4], o[5]); u.w = pack_bf16x2(o[6], o[7]);
            stg_v4(p.y + row * H + ch * 8, u);
        }
    }
}

template <int NC>
__global__ void __launch_bounds__(kEmbWarps * 32) embed_fwd_kernel(const EmbedParams p) { embed_fwd_body<NC, false>(p); }
template <int NC>
__global__ void __launch_bounds__(kEmbWarps * 32) embed_fwd_off_kernel(const EmbedParams p) { embed_fwd_body<NC, true>(p); }

// Adjoint of the gather / concat: word rows are scattered with vector reductions; the position, token-type and visual
// position / type gradients — a few rows that EVERY example adds into — are first summed in registers over a chunk of
// examples at a fixed sequence position (a warp task = (position s, 32 examples)), so each table row receives one vector
// reduction per task instead of one scalar atomic per element (which made atomic contention the bulk of the kernel's time).
// smem: [n_types][H] text types, [n_types][H] visual types, [H] visual position row 0 (block accumulators, flushed once)
// FROZEN (embed_bwd_frozen_kernel): some gradient tables are NULL (frozen); they receive nothing.
template <int NC, bool FROZEN>
__device__ __forceinline__ void embed_bwd_body(const EmbedBwdParams& p, int cb, int nb) {
    extern __shared__ float acc[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int H = p.H, chunks = H >> 3, S = p.T + p.V, nt = p.n_types;
    const int nacc = (2 * nt + 1) * H;
    for (int i = threadIdx.x; i < nacc; i += blockDim.x) acc[i] = 0.f;
    __syncthreads();
    const int tasks = S * nb;
    for (int task = blockIdx.x * kEmbWarps + warp; task < tasks; task += gridDim.x * kEmbWarps) {
        const int s = task % S, bc = task / S;
        const int b0 = bc * cb, b1 = min(p.B, b0 + cb);
        const bool text = s < p.T;
        float psum[NC][8], t0[NC][8], t1[NC][8];   // position row, token types 0 / 1 (other types: shared-memory atomics)
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
            for (int i = 0; i < 8; ++i) psum[c][i] = t0[c][i] = t1[c][i] = 0.f;
        for (int b = b0; b < b1; ++b) {
            const long long row = static_cast<long long>(b) * S + s;
            float* g0 = nullptr;
            bf16* dv = nullptr;
            int ty;
            if (text) {
                if (!FROZEN || p.dword != nullptr)
                    g0 = p.dword + static_cast<long long>(clampi(p.ids[static_cast<long long>(b) * p.T + s], p.vocab)) * H;
                ty = clampi(p.tt[static_cast<long long>(b) * p.T + s], nt);
            } else {
                dv = p.dvis + (static_cast<long long>(b) * p.V + (s - p.T)) * H;
                ty = clampi(p.vt[static_cast<long long>(b) * p.V + (s - p.T)], nt);
            }
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                const int ch = lane + c * 32;
                if (ch < chunks) {
                    const uint4 u = ldg_v4(p.de + row * H + ch * 8);
                    if (dv != nullptr) stg_v4(dv + ch * 8, u);
                    const float2 x0 = unpack_bf16x2(u.x), x1 = unpack_bf16x2(u.y), x2 = unpack_bf16x2(u.z), x3 = unpack_bf16x2(u.w);
                    const float d[8] = {x0.x, x0.y, x1.x, x1.y, x2.x, x2.y, x3.x, x3.y};
                    if (g0 != nullptr) {
                        red_add_v4_f32(g0 + ch * 8, d[0], d[1], d[2], d[3]);
                        red_add_v4_f32(g0 + ch * 8 + 4, d[4], d[5], d[6], d[7]);
                    }
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        psum[c][i] += d[i];
                        if (ty == 0) t0[c][i] += d[i];
                        else if (ty == 1) t1[c][i] += d[i];
                        else atomicAdd(acc + ((text ? 0 : nt) + ty) * H + ch * 8 + i, d[i]);
                    }
                }
            }
        }
        // flush the task: position row (text: global table row s; visual: the block's accumulator of visual position 0), types
        float* prow = text && (!FROZEN || p.dpos != nullptr) ? p.dpos + static_cast<long long>(s < p.max_pos ? s : p.max_pos - 1) * H
                                                              : nullptr;
        float* a0 = acc + (text ? 0 : nt) * H;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int ch = lane + c * 32;
            if (ch < chunks) {
                if (prow != nullptr) {
                    red_add_v4_f32(prow + ch * 8, psum[c][0], psum[c][1], psum[c][2], psum[c][3]);
                    red_add_v4_f32(prow + ch * 8 + 4, psum[c][4], psum[c][5], psum[c][6], psum[c][7]);
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    if (FROZEN ? !text : prow == nullptr) atomicAdd(acc + 2 * nt * H + ch * 8 + i, psum[c][i]);
                    atomicAdd(a0 + ch * 8 + i, t0[c][i]);
                    if (nt > 1) atomicAdd(a0 + H + ch * 8 + i, t1[c][i]);
                }
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nt * H; i += blockDim.x) {
        if (!FROZEN || p.dtype != nullptr) atomicAdd(p.dtype + i, acc[i]);
        if (!FROZEN || p.dtype_vis != nullptr) atomicAdd(p.dtype_vis + i, acc[nt * H + i]);
    }
    if (!FROZEN || p.dpos_vis != nullptr)
        for (int i = threadIdx.x; i < H; i += blockDim.x) atomicAdd(p.dpos_vis + i, acc[2 * nt * H + i]);
}
template <int NC>
__global__ void __launch_bounds__(kEmbWarps * 32) embed_bwd_kernel(const EmbedBwdParams p, int cb, int nb) {
    embed_bwd_body<NC, false>(p, cb, nb);
}
template <int NC>
__global__ void __launch_bounds__(kEmbWarps * 32, 1) embed_bwd_frozen_kernel(const EmbedBwdParams p, int cb, int nb) {
    embed_bwd_body<NC, true>(p, cb, nb);
}

__global__ void mask_bias_kernel(const long long* __restrict__ input_mask, const long long* __restrict__ image_mask,
                                 float* __restrict__ out, int B, int T, int V) {
    const int S = T + V;
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<long long>(B) * S) return;
    const int b = static_cast<int>(i / S), s = static_cast<int>(i % S);
    const long long m = s < T ? input_mask[static_cast<long long>(b) * T + s]
                              : (image_mask ? image_mask[static_cast<long long>(b) * V + (s - T)] : 1);
    out[i] = (1.0f - static_cast<float>(m)) * -10000.0f;
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n8) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(src) + 2 * i);
        const float4 b = __ldg(reinterpret_cast<const float4*>(src) + 2 * i + 1);
        uint4 u;
        u.x = pack_bf16x2(a.x, a.y); u.y = pack_bf16x2(a.z, a.w);
        u.z = pack_bf16x2(b.x, b.y); u.w = pack_bf16x2(b.z, b.w);
        reinterpret_cast<uint4*>(dst)[i] = u;
    }
}
__global__ void cast_bf16_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, long long n8) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(src) + i);
        const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
        reinterpret_cast<float4*>(dst)[2 * i] = make_float4(a.x, a.y, b.x, b.y);
        reinterpret_cast<float4*>(dst)[2 * i + 1] = make_float4(c.x, c.y, d.x, d.y);
    }
}

// out[N] += column sums of x[M, N] (bf16). block = 32 x 8: x -> 8-column chunk, y -> row phase; four rows per
// iteration so every thread keeps 4 x 16 B loads in flight (the kernel is pure HBM streaming). The rows are swept from the
// LAST to the first: the tensor was just written by the previous kernel, whose tiles run in increasing row order, so its tail
// is what the L2 still holds.
// PART = true (deterministic mode): out is the workspace and block row y STORES its sums to out[y * N + col]; partials_reduce
// adds them in blockIdx.y order.
template <bool PART>
__device__ __forceinline__ void colsum_body(const bf16* __restrict__ x, long long ld, float* __restrict__ out, int M, int N) {
    __shared__ float red[8][32][9];
    const int ch = blockIdx.x * 32 + threadIdx.x;
    pdl_trigger();
    pdl_wait();
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (ch * 8 < N) {
        const int stride = gridDim.y * 8;
        int r = blockIdx.y * 8 + threadIdx.y;
        for (; r + 3 * stride < M; r += 4 * stride) {
            uint4 u[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) u[j] = ldg_v4(x + static_cast<long long>(M - 1 - (r + j * stride)) * ld + ch * 8);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 x0 = unpack_bf16x2(u[j].x), x1 = unpack_bf16x2(u[j].y), x2 = unpack_bf16x2(u[j].z), x3 = unpack_bf16x2(u[j].w);
                a[0] += x0.x; a[1] += x0.y; a[2] += x1.x; a[3] += x1.y; a[4] += x2.x; a[5] += x2.y; a[6] += x3.x; a[7] += x3.y;
            }
        }
        for (; r < M; r += stride) {
            const uint4 u = ldg_v4(x + static_cast<long long>(M - 1 - r) * ld + ch * 8);
            const float2 x0 = unpack_bf16x2(u.x), x1 = unpack_bf16x2(u.y), x2 = unpack_bf16x2(u.z), x3 = unpack_bf16x2(u.w);
            a[0] += x0.x; a[1] += x0.y; a[2] += x1.x; a[3] += x1.y; a[4] += x2.x; a[5] += x2.y; a[6] += x3.x; a[7] += x3.y;
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) red[threadIdx.y][threadIdx.x][i] = a[i];
    __syncthreads();
    if (threadIdx.y == 0 && ch * 8 < N) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float s = 0.f;
#pragma unroll
            for (int y = 0; y < 8; ++y) s += red[y][threadIdx.x][i];
            if constexpr (PART) out[static_cast<long long>(blockIdx.y) * N + ch * 8 + i] = s;
            else atomicAdd(out + ch * 8 + i, s);
        }
    }
}
__global__ void __launch_bounds__(256)
colsum_kernel(const bf16* __restrict__ x, long long ld, float* __restrict__ out, int M, int N) { colsum_body<false>(x, ld, out, M, N); }
__global__ void __launch_bounds__(256)
colsum_part_kernel(const bf16* __restrict__ x, long long ld, float* __restrict__ out, int M, int N) { colsum_body<true>(x, ld, out, M, N); }

// ---- embedding backward in deterministic mode --------------------------------------------------------------------------------
// Every table row the backward adds into is a KEY in one key space: word rows [0, vocab), position rows [vocab, + max_pos), text
// types [.., + n_types), visual position 0 (one key), visual types [.., + n_types). Each text row contributes three (key, row)
// items (word, position, type), each visual row two (visual position 0, visual type), listed in row order. A stable radix sort
// by key makes every key's items one run, in row order. The run sums are then formed in a fixed association: the sorted items
// are cut into windows of kSegWin; embed_seg_kernel sums each run's items inside a window in order and adds a run that lies
// inside one window straight into its table row (no other writer has that key), or stores the partial of a run that crosses a
// window edge (its head part in a window it did not start in, its tail part in the window it started in); embed_seg_join_kernel
// adds those partials in window order for the window a crossing run started in, and adds the sum into the table row once.
constexpr int kSegWin = 64;

__device__ __forceinline__ float* embed_key_row(const EmbedBwdParams& p, unsigned k) {
    const long long H = p.H;
    if (k < static_cast<unsigned>(p.vocab)) return p.dword ? p.dword + k * H : nullptr;
    k -= p.vocab;
    if (k < static_cast<unsigned>(p.max_pos)) return p.dpos ? p.dpos + k * H : nullptr;
    k -= p.max_pos;
    if (k < static_cast<unsigned>(p.n_types)) return p.dtype ? p.dtype + k * H : nullptr;
    k -= p.n_types;
    if (k == 0) return p.dpos_vis;
    return p.dtype_vis ? p.dtype_vis + (k - 1) * H : nullptr;
}

// one thread per row of de: its (key, row) items; the visual rows are also copied to dvis (the projection's weight-gradient input)
__global__ void __launch_bounds__(256) embed_keys_kernel(const EmbedBwdParams p, unsigned* __restrict__ keys, int* __restrict__ vals) {
    const int S = p.T + p.V;
    const long long row = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (row >= static_cast<long long>(p.B) * S) return;
    const int b = static_cast<int>(row / S), s = static_cast<int>(row % S);
    const unsigned kpos = p.vocab, ktype = kpos + p.max_pos, kvpos = ktype + p.n_types;
    if (s < p.T) {
        const long long i = (static_cast<long long>(b) * p.T + s) * 3, t = static_cast<long long>(b) * p.T + s;
        keys[i] = clampi(p.ids[t], p.vocab);
        keys[i + 1] = kpos + (s < p.max_pos ? s : p.max_pos - 1);
        keys[i + 2] = ktype + clampi(p.tt[t], p.n_types);
        vals[i] = vals[i + 1] = vals[i + 2] = static_cast<int>(row);
    } else {
        const long long t = static_cast<long long>(b) * p.V + (s - p.T), i = 3LL * p.B * p.T + 2 * t;
        keys[i] = kvpos;
        keys[i + 1] = kvpos + 1 + clampi(p.vt[t], p.n_types);
        vals[i] = vals[i + 1] = static_cast<int>(row);
    }
}

__global__ void __launch_bounds__(256) embed_vis_copy_kernel(const EmbedBwdParams p) {
    const int S = p.T + p.V, c8 = p.H / 8;
    const long long n = static_cast<long long>(p.B) * p.V * c8;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long r = i / c8, c = i - r * c8;
        const long long b = r / p.V, v = r - b * p.V;
        stg_v4(p.dvis + r * p.H + c * 8, ldg_v4(p.de + (b * S + p.T + v) * p.H + c * 8));
    }
}

template <int NC>
__device__ __forceinline__ void seg_add_row(const EmbedBwdParams& p, int row, int lane, float (&acc)[NC][8]) {
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        const int ch = lane + c * 32;
        if (ch < p.H / 8) {
            const uint4 u = ldg_v4(p.de + static_cast<long long>(row) * p.H + ch * 8);
            const float2 x0 = unpack_bf16x2(u.x), x1 = unpack_bf16x2(u.y), x2 = unpack_bf16x2(u.z), x3 = unpack_bf16x2(u.w);
            acc[c][0] += x0.x; acc[c][1] += x0.y; acc[c][2] += x1.x; acc[c][3] += x1.y;
            acc[c][4] += x2.x; acc[c][5] += x2.y; acc[c][6] += x3.x; acc[c][7] += x3.y;
        }
    }
}
template <int NC>
__device__ __forceinline__ void seg_flush(float* dst, bool add, int H, int lane, float (&acc)[NC][8]) {
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        const int ch = lane + c * 32;
        if (ch < H / 8) {
            float4* d = reinterpret_cast<float4*>(dst + ch * 8);
            float4 a0 = make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]), a1 = make_float4(acc[c][4], acc[c][5], acc[c][6], acc[c][7]);
            if (add) {
                const float4 o0 = d[0], o1 = d[1];
                a0.x += o0.x; a0.y += o0.y; a0.z += o0.z; a0.w += o0.w;
                a1.x += o1.x; a1.y += o1.y; a1.z += o1.z; a1.w += o1.w;
            }
            d[0] = a0; d[1] = a1;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;
    }
}

// one warp per window; slots: [2][windows][H] fp32 (0: head partials, 1: tail partials)
// FROZEN: some tables are NULL (frozen). Their items stay in the sort, so every window and sum order is that of the full call,
// but their runs are neither summed nor flushed.
template <int NC, bool FROZEN = false>
__global__ void __launch_bounds__(kEmbWarps * 32)
embed_seg_kernel(const EmbedBwdParams p, const unsigned* __restrict__ keys, const int* __restrict__ vals, int n, float* __restrict__ slots) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kEmbWarps + warp, windows = (n + kSegWin - 1) / kSegWin;
    if (w >= windows) return;
    const int beg = w * kSegWin, end = min(beg + kSegWin, n);
    const bool from_before = beg > 0 && keys[beg - 1] == keys[beg];
    float acc[NC][8];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;
    int run_beg = beg;
    for (int i = beg; i < end; ++i) {
        const unsigned k = keys[i];
        if constexpr (FROZEN) {
            if (embed_key_row(p, k) == nullptr) { run_beg = i + 1; continue; }
        }
        seg_add_row<NC>(p, vals[i], lane, acc);
        const bool run_end = i + 1 == n || keys[i + 1] != k;
        if (run_end || i + 1 == end) {
            const bool head = run_beg == beg && from_before;
            if (head) seg_flush<NC>(slots + static_cast<long long>(w) * p.H, false, p.H, lane, acc);
            else if (!run_end) seg_flush<NC>(slots + (static_cast<long long>(windows) + w) * p.H, false, p.H, lane, acc);
            else seg_flush<NC>(embed_key_row(p, k), true, p.H, lane, acc);
            run_beg = i + 1;
        }
    }
}

// one warp per window: the window a crossing run started in adds its tail partial and the head partials of the following windows
template <int NC, bool FROZEN = false>
__global__ void __launch_bounds__(kEmbWarps * 32)
embed_seg_join_kernel(const EmbedBwdParams p, const unsigned* __restrict__ keys, int n, const float* __restrict__ slots) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kEmbWarps + warp, windows = (n + kSegWin - 1) / kSegWin;
    if (w >= windows) return;
    const int beg = w * kSegWin, end = min(beg + kSegWin, n);
    const unsigned k = keys[end - 1];
    const bool starts_here = !(beg > 0 && keys[beg - 1] == k && keys[beg] == k);
    if (!starts_here || end == n || keys[end] != k) return;
    if constexpr (FROZEN) {
        if (embed_key_row(p, k) == nullptr) return;
    }
    float acc[NC][8];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;
    auto add_slot = [&](const float* src) {
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int ch = lane + c * 32;
            if (ch < p.H / 8) {
                const float4 a = *reinterpret_cast<const float4*>(src + ch * 8), b = *reinterpret_cast<const float4*>(src + ch * 8 + 4);
                acc[c][0] += a.x; acc[c][1] += a.y; acc[c][2] += a.z; acc[c][3] += a.w;
                acc[c][4] += b.x; acc[c][5] += b.y; acc[c][6] += b.z; acc[c][7] += b.w;
            }
        }
    };
    add_slot(slots + (static_cast<long long>(windows) + w) * p.H);
    for (int w2 = w + 1; w2 < windows; ++w2) {
        add_slot(slots + static_cast<long long>(w2) * p.H);
        const int e2 = min((w2 + 1) * kSegWin, n);
        if (e2 == n || keys[e2] != k) break;
    }
    seg_flush<NC>(embed_key_row(p, k), true, p.H, lane, acc);
}

static long long embed_items(int B, int T, int V) { return 3LL * B * T + 2LL * B * V; }
static long long al256(long long x) { return (x + 255) / 256 * 256; }
long long embed_sort_temp_bytes(int B, int T, int V) {
    size_t bytes = 0;
    cub::DoubleBuffer<unsigned> k(nullptr, nullptr);
    cub::DoubleBuffer<int> v(nullptr, nullptr);
    if (cub::DeviceRadixSort::SortPairs(nullptr, bytes, k, v, static_cast<int>(embed_items(B, T, V)), 0, 32) != cudaSuccess) return -1;
    return static_cast<long long>(bytes);
}
// workspace layout: keys[2][n] (u32), vals[2][n] (i32), slots [2][windows][H] fp32, sort temp. sort_temp < 0: a bound on the sort's
// temporary storage (32 bytes per item + 1 MB, several times what the radix sort takes) for vb_deterministic_workspace_bytes,
// which must work without a device
long long embed_bwd_det_bytes(int B, int T, int V, int H, long long sort_temp) {
    const long long n = embed_items(B, T, V), windows = (n + kSegWin - 1) / kSegWin;
    if (sort_temp < 0) sort_temp = 32 * n + (1 << 20);
    return 4 * al256(4 * n) + al256(2 * windows * H * 4) + al256(sort_temp);
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
int embed_fwd(const EmbedParams& p, cudaStream_t st) {
    VB_REQUIRE(p.H % 8 == 0 && p.H <= 1024, "embed: H=%d must be a multiple of 8 and <= 1024", p.H);
    VB_REQUIRE(p.B > 0 && p.T > 0 && p.V >= 0, "embed: bad shape");
    VB_REQUIRE(p.T <= p.max_pos, "embed: text length %d exceeds max_position_embeddings %d", p.T, p.max_pos);
    const long long rows = static_cast<long long>(p.B) * (p.T + p.V);
    const int grid = static_cast<int>((rows + kEmbWarps - 1) / kEmbWarps);
    const int nc = (p.H / 8 + 31) / 32;
    ProfScope ps(st, PROF_EMBED, 8.0 * rows * p.H, 1);
    if (p.drop_offset != nullptr) {   // dropout seed + *offset, read by the kernel (vb_set_dropout_offset)
        switch (nc) {
            case 1: embed_fwd_off_kernel<1><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
            case 2: embed_fwd_off_kernel<2><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
            case 3: embed_fwd_off_kernel<3><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
            default: embed_fwd_off_kernel<4><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
        }
    } else {
        switch (nc) {
            case 1: embed_fwd_kernel<1><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
            case 2: embed_fwd_kernel<2><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
            case 3: embed_fwd_kernel<3><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
            default: embed_fwd_kernel<4><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
        }
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static int embed_bwd_det(const EmbedBwdParams& p, const DetWs& det, cudaStream_t st) {
    VB_REQUIRE(((reinterpret_cast<uintptr_t>(p.dtype) | reinterpret_cast<uintptr_t>(p.dpos_vis) | reinterpret_cast<uintptr_t>(p.dtype_vis)) & 15) == 0,
               "embed backward: gradient tables must be 16-byte aligned");
    const long long n = embed_items(p.B, p.T, p.V), windows = (n + kSegWin - 1) / kSegWin;
    VB_REQUIRE(n < (1LL << 31) && static_cast<long long>(p.vocab) + p.max_pos + 2LL * p.n_types + 1 < (1LL << 32),
               "embed backward: too many rows / table rows for deterministic mode");
    const long long temp = embed_sort_temp_bytes(p.B, p.T, p.V);
    VB_REQUIRE(temp >= 0, "embed backward: radix sort size query failed");
    VB_TRY_RC(det_require(embed_bwd_det_bytes(p.B, p.T, p.V, p.H, temp), "embed backward"));
    char* ws = static_cast<char*>(det.ptr);
    unsigned* k0 = reinterpret_cast<unsigned*>(ws);
    unsigned* k1 = reinterpret_cast<unsigned*>(ws + al256(4 * n));
    int* v0 = reinterpret_cast<int*>(ws + 2 * al256(4 * n));
    int* v1 = reinterpret_cast<int*>(ws + 3 * al256(4 * n));
    float* slots = reinterpret_cast<float*>(ws + 4 * al256(4 * n));
    void* sort_temp = ws + 4 * al256(4 * n) + al256(2 * windows * p.H * 4);
    const long long rows = static_cast<long long>(p.B) * (p.T + p.V);
    const unsigned max_key = static_cast<unsigned>(p.vocab + p.max_pos + 2 * p.n_types);
    int end_bit = 1;
    while (end_bit < 32 && (max_key >> end_bit) != 0) ++end_bit;
    const int nc = (p.H / 8 + 31) / 32;
    const int seg_grid = static_cast<int>((windows + kEmbWarps - 1) / kEmbWarps);
    ProfScope ps(st, PROF_EMBED, 6.0 * rows * p.H, 5);
    embed_keys_kernel<<<static_cast<int>((rows + 255) / 256), 256, 0, st>>>(p, k0, v0);
    VB_CHECK_CUDA(cudaGetLastError());
    if (p.V > 0) {
        long long blocks = (static_cast<long long>(p.B) * p.V * (p.H / 8) + 255) / 256;
        if (blocks > num_sms() * 8) blocks = num_sms() * 8;
        embed_vis_copy_kernel<<<static_cast<int>(blocks), 256, 0, st>>>(p);
        VB_CHECK_CUDA(cudaGetLastError());
    }
    cub::DoubleBuffer<unsigned> kb(k0, k1);
    cub::DoubleBuffer<int> vb(v0, v1);
    size_t tb = static_cast<size_t>(temp);
    VB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(sort_temp, tb, kb, vb, static_cast<int>(n), 0, end_bit, st));
    const unsigned* keys = kb.Current();
    const int* vals = vb.Current();
#define VB_SEG(NC, F)                                                                                                     \
    embed_seg_kernel<NC, F><<<seg_grid, kEmbWarps * 32, 0, st>>>(p, keys, vals, static_cast<int>(n), slots);             \
    embed_seg_join_kernel<NC, F><<<seg_grid, kEmbWarps * 32, 0, st>>>(p, keys, static_cast<int>(n), slots)
    const bool frozen = !p.dword || !p.dpos || !p.dtype || !p.dpos_vis || !p.dtype_vis;
    switch (nc) {
        case 1: if (frozen) { VB_SEG(1, true); } else { VB_SEG(1, false); } break;
        case 2: if (frozen) { VB_SEG(2, true); } else { VB_SEG(2, false); } break;
        case 3: if (frozen) { VB_SEG(3, true); } else { VB_SEG(3, false); } break;
        default: if (frozen) { VB_SEG(4, true); } else { VB_SEG(4, false); } break;
    }
#undef VB_SEG
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int embed_bwd(const EmbedBwdParams& p, cudaStream_t st) {
    VB_REQUIRE(p.H % 8 == 0 && p.H <= 1024, "embed backward: H=%d must be a multiple of 8 and <= 1024", p.H);
    VB_REQUIRE((reinterpret_cast<uintptr_t>(p.dword) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.dpos) & 15) == 0,
               "embed backward: gradient tables must be 16-byte aligned");
    const DetWs det = det_ws();
    if (det.ptr != nullptr) return embed_bwd_det(p, det, st);
    const bool frozen = !p.dword || !p.dpos || !p.dtype || !p.dpos_vis || !p.dtype_vis;
    if (!p.dword && !p.dpos && !p.dtype && !p.dpos_vis && !p.dtype_vis && p.V == 0) return 0;   // nothing to scatter or copy
    const long long rows = static_cast<long long>(p.B) * (p.T + p.V);
    const int cb = p.B < 32 ? p.B : 32, nb = (p.B + cb - 1) / cb;   // a warp task: one sequence position, up to 32 examples
    const long long tasks = static_cast<long long>(p.T + p.V) * nb;
    int grid = num_sms() * 2;
    const long long need = (tasks + kEmbWarps - 1) / kEmbWarps;
    if (grid > need) grid = static_cast<int>(need);
    const size_t smem = static_cast<size_t>(2 * p.n_types + 1) * p.H * sizeof(float);
    VB_REQUIRE(smem <= 48 * 1024, "embed backward: type_vocab_size * hidden too large for shared memory");
    const int nc = (p.H / 8 + 31) / 32;
    {
        ProfScope ps(st, PROF_EMBED, 6.0 * rows * p.H, 1);
        if (frozen) {
            switch (nc) {
                case 1: embed_bwd_frozen_kernel<1><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
                case 2: embed_bwd_frozen_kernel<2><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
                case 3: embed_bwd_frozen_kernel<3><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
                default: embed_bwd_frozen_kernel<4><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
            }
        } else {
            switch (nc) {
                case 1: embed_bwd_kernel<1><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
                case 2: embed_bwd_kernel<2><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
                case 3: embed_bwd_kernel<3><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
                default: embed_bwd_kernel<4><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
            }
        }
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int mask_bias(const long long* input_mask, const long long* image_mask, float* out, int B, int T, int V, cudaStream_t st) {
    const long long n = static_cast<long long>(B) * (T + V);
    VB_REQUIRE(n > 0, "mask_bias: empty");
    {
        ProfScope ps(st, PROF_OTHER, 12.0 * n, 1);
        mask_bias_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, st>>>(input_mask, image_mask, out, B, T, V);
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int cast_f32_bf16(const float* src, void* dst, long long n, cudaStream_t st) {
    VB_REQUIRE(n % 8 == 0, "cast: element count must be a multiple of 8");
    VB_REQUIRE(all_aligned16(src, dst), "cast: src and dst must be 16-byte aligned");
    if (n == 0) return 0;
    const long long n8 = n / 8;
    long long blocks = (n8 + 255) / 256;
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    {
        ProfScope ps(st, PROF_OTHER, 6.0 * n, 1);
        cast_f32_bf16_kernel<<<static_cast<int>(blocks), 256, 0, st>>>(src, static_cast<bf16*>(dst), n8);
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
int cast_bf16_f32(const void* src, float* dst, long long n, cudaStream_t st) {
    VB_REQUIRE(n % 8 == 0, "cast: element count must be a multiple of 8");
    VB_REQUIRE(all_aligned16(src, dst), "cast: src and dst must be 16-byte aligned");
    if (n == 0) return 0;
    const long long n8 = n / 8;
    long long blocks = (n8 + 255) / 256;
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    {
        ProfScope ps(st, PROF_OTHER, 6.0 * n, 1);
        cast_bf16_f32_kernel<<<static_cast<int>(blocks), 256, 0, st>>>(static_cast<const bf16*>(src), dst, n8);
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static int colsum_gy(int M, int N) {
    const int gx = (N / 8 + 31) / 32;
    int gy = (num_sms() * 6) / gx;
    if (gy < 1) gy = 1;
    if (gy > (M + 7) / 8) gy = (M + 7) / 8;
    return gy;
}
long long colsum_det_bytes(int M, int N) { return static_cast<long long>(colsum_gy(M, N)) * N * 4; }

int colsum(const void* x, long long ld, float* out, int M, int N, cudaStream_t st) {
    VB_REQUIRE(N % 8 == 0 && M > 0, "colsum: bad shape");
    VB_REQUIRE(ld >= N && ld % 8 == 0, "colsum: ld=%lld must be a multiple of 8 and >= N=%d", ld, N);
    VB_REQUIRE(x && out && all_aligned16(x), "colsum: x must be 16-byte aligned and out not NULL");
    const int gx = (N / 8 + 31) / 32;
    const int gy = colsum_gy(M, N);
    const DetWs det = det_ws();
    if (det.ptr != nullptr) {
        VB_TRY_RC(det_require(colsum_det_bytes(M, N), "colsum"));
        {
            ProfScope ps(st, PROF_COLSUM, 2.0 * M * N, 1);
            VB_CHECK_CUDA(launch_pdl(colsum_part_kernel, dim3(gx, gy), dim3(32, 8), 0, st, static_cast<const bf16*>(x), ld,
                                     static_cast<float*>(det.ptr), M, N));
        }
        VB_CHECK_CUDA(cudaGetLastError());
        return partials_reduce(static_cast<const float*>(det.ptr), gy, N, N, out, nullptr, nullptr, st);
    }
    {
        ProfScope ps(st, PROF_COLSUM, 2.0 * M * N, 1);
        VB_CHECK_CUDA(launch_pdl(colsum_kernel, dim3(gx, gy), dim3(32, 8), 0, st, static_cast<const bf16*>(x), ld, out, M, N));
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace vb
