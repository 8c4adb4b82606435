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
#include "vb_internal.h"

namespace vb {

constexpr int kEmbWarps = 8;

__device__ __forceinline__ int clampi(long long v, int hi) { return v < 0 ? 0 : (v >= hi ? hi - 1 : static_cast<int>(v)); }

template <int NC>
__global__ void __launch_bounds__(kEmbWarps * 32)
embed_fwd_kernel(const EmbedParams p) {
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
                const uint32_t keep = dropout_keep8(p.drop_seed, p.drop_stream, e8, p.drop_thresh16);
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

// Adjoint of the gather / concat: word rows are scattered with vector reductions; the position, token-type and visual
// position / type gradients — a few rows that EVERY example adds into — are first summed in registers over a chunk of
// examples at a fixed sequence position (a warp task = (position s, 32 examples)), so each table row receives one vector
// reduction per task instead of one scalar atomic per element (which made atomic contention the bulk of the kernel's time).
// smem: [n_types][H] text types, [n_types][H] visual types, [H] visual position row 0 (block accumulators, flushed once)
template <int NC>
__global__ void __launch_bounds__(kEmbWarps * 32)
embed_bwd_kernel(const EmbedBwdParams p, int cb, int nb) {
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
        float* prow = text ? p.dpos + static_cast<long long>(s < p.max_pos ? s : p.max_pos - 1) * H : nullptr;
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
                    if (prow == nullptr) atomicAdd(acc + 2 * nt * H + ch * 8 + i, psum[c][i]);
                    atomicAdd(a0 + ch * 8 + i, t0[c][i]);
                    if (nt > 1) atomicAdd(a0 + H + ch * 8 + i, t1[c][i]);
                }
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nt * H; i += blockDim.x) {
        atomicAdd(p.dtype + i, acc[i]);
        atomicAdd(p.dtype_vis + i, acc[nt * H + i]);
    }
    for (int i = threadIdx.x; i < H; i += blockDim.x) atomicAdd(p.dpos_vis + i, acc[2 * nt * H + i]);
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
__global__ void __launch_bounds__(256)
colsum_kernel(const bf16* __restrict__ x, long long ld, float* __restrict__ out, int M, int N) {
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
            atomicAdd(out + ch * 8 + i, s);
        }
    }
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
    switch (nc) {
        case 1: embed_fwd_kernel<1><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
        case 2: embed_fwd_kernel<2><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
        case 3: embed_fwd_kernel<3><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
        default: embed_fwd_kernel<4><<<grid, kEmbWarps * 32, 0, st>>>(p); break;
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int embed_bwd(const EmbedBwdParams& p, cudaStream_t st) {
    VB_REQUIRE(p.H % 8 == 0 && p.H <= 1024, "embed backward: H=%d must be a multiple of 8 and <= 1024", p.H);
    VB_REQUIRE((reinterpret_cast<uintptr_t>(p.dword) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.dpos) & 15) == 0,
               "embed backward: gradient tables must be 16-byte aligned");
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
        switch (nc) {
            case 1: embed_bwd_kernel<1><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
            case 2: embed_bwd_kernel<2><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
            case 3: embed_bwd_kernel<3><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
            default: embed_bwd_kernel<4><<<grid, kEmbWarps * 32, smem, st>>>(p, cb, nb); break;
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

int colsum(const void* x, long long ld, float* out, int M, int N, cudaStream_t st) {
    VB_REQUIRE(N % 8 == 0 && M > 0, "colsum: bad shape");
    const int gx = (N / 8 + 31) / 32;
    int gy = (num_sms() * 6) / gx;
    if (gy < 1) gy = 1;
    if (gy > (M + 7) / 8) gy = (M + 7) / 8;
    {
        ProfScope ps(st, PROF_COLSUM, 2.0 * M * N, 1);
        VB_CHECK_CUDA(launch_pdl(colsum_kernel, dim3(gx, gy), dim3(32, 8), 0, st, static_cast<const bf16*>(x), ld, out, M, N));
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace vb
