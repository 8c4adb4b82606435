// vb_layernorm.cu — BertLayerNorm forward / backward (reference modeling.py:162-175: TF style,
// biased variance, eps inside the sqrt, statistics in fp32) for bf16 activations.
//
// HBM-bound row kernels: one warp per row, the row lives in registers (16-byte loads, lane l owns
// column chunks l, l+32, ...), warp-shuffle reductions, no shared memory in forward. Backward also
// produces the column reductions a fused residual block needs in the same pass: dgamma, dbeta and
// the bias gradient of the Linear that precedes the LayerNorm (column sum of the output gradient),
// accumulated in registers across a grid-stride row loop, reduced through shared memory and flushed
// with one fp32 atomic per column per block.
#include "../../include/vbert_b200.h"
#include "vb_common.cuh"

namespace vb {

constexpr int kLnWarps = 8;

template <int NC>
__global__ void __launch_bounds__(kLnWarps * 32)
ln_fwd_kernel(const bf16* __restrict__ x, long long ldx, const float* __restrict__ gamma,
              const float* __restrict__ beta, bf16* __restrict__ y, long long ldy, float* __restrict__ mean_out,
              float* __restrict__ rstd_out, int rows, int H, float eps) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = blockIdx.x * kLnWarps + warp;
    pdl_trigger();
    pdl_wait();
    if (row >= rows) return;
    const int chunks = H >> 3;
    float v[NC][8];
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        const int ch = lane + c * 32;
        if (ch < chunks) {
            const uint4 u = ldg_v4(x + row * ldx + ch * 8);
            const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), d = unpack_bf16x2(u.z), e = unpack_bf16x2(u.w);
            v[c][0] = a.x; v[c][1] = a.y; v[c][2] = b.x; v[c][3] = b.y;
            v[c][4] = d.x; v[c][5] = d.y; v[c][6] = e.x; v[c][7] = e.y;
#pragma unroll
            for (int i = 0; i < 8; ++i) s += v[c][i];
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[c][i] = 0.f;
        }
    }
    const float mean = warp_sum(s) / H;
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        if (lane + c * 32 < chunks) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { const float d = v[c][i] - mean; q += d * d; }
        }
    }
    const float rstd = rsqrtf(warp_sum(q) / H + eps);
    if (lane == 0) {
        if (mean_out) mean_out[row] = mean;
        if (rstd_out) rstd_out[row] = rstd;
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        const int ch = lane + c * 32;
        if (ch < chunks) {
            const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + ch * 8));
            const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + ch * 8 + 4));
            const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + ch * 8));
            const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + ch * 8 + 4));
            const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            float o[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = g[i] * ((v[c][i] - mean) * rstd) + b[i];
            uint4 u;
            u.x = pack_bf16x2(o[0], o[1]); u.y = pack_bf16x2(o[2], o[3]);
            u.z = pack_bf16x2(o[4], o[5]); u.w = pack_bf16x2(o[6], o[7]);
            stg_v4(y + row * ldy + ch * 8, u);
        }
    }
}

// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * gamma,  xhat = (x - mean) * rstd
// dgamma += sum_rows dy * xhat ; dbeta += sum_rows dy ; dbias += sum_rows dx_out
// where dx_out = dx (no dropout) or dx * keep / (1-p) (the gradient entering the preceding Linear
// when its output went through dropout before the residual add; dx itself continues down the
// residual branch).
//
// Nominally HBM-bound, in practice instruction-issue bound (IPC 2.5, ~50 % of HBM peak): the row is unpacked once and
// xhat / dy stay in fp32 registers for both passes; gamma and the three column accumulators live in shared memory (one
// private slab per warp: plain float4 read-modify-write, no atomics, no bank conflicts thanks to the split lo/hi
// float4 layout); 123 registers, 2 blocks (16 warps) per SM.
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    uint4 u;
    u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
    u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
    return u;
}
// float4 slot of (array a, chunk ch, half h) inside a slab of `chunks` chunks: lanes -> consecutive 16 B
__device__ __forceinline__ int slot(int a, int h, int ch, int chunks) { return (a * 2 + h) * chunks + ch; }

// PART = false: the block's column sums go to dgamma / dbeta / dbias by atomicAdd. PART = true (deterministic mode): dgamma is
// the workspace and block b STORES its sums to dgamma[(b * 3 + array) * H + col]; partials_reduce adds them in block order.
// OFF = true (vb_set_dropout_offset): the dropout seed is drop_seed + *drop_offset, read once global memory may be touched.
// SUMS = false (a caller whose dgamma, dbeta and dbias are all frozen): a pure row pass — dx and dx_drop only, no shared-memory
// accumulators, no atomics and no partial stores; PART is then meaningless and dgamma / dbeta / dbias are not read.
template <int NC, bool PART, bool OFF = false, bool SUMS = true>
__device__ __forceinline__ void
ln_bwd_body(const bf16* __restrict__ dy, const bf16* __restrict__ x, const float* __restrict__ mean,
            const float* __restrict__ rstd, const float* __restrict__ gamma, bf16* __restrict__ dx,
            bf16* __restrict__ dx_drop, float* __restrict__ dgamma, float* __restrict__ dbeta,
            float* __restrict__ dbias, int rows, int H, float drop_scale, unsigned drop_thresh16,
            unsigned long long drop_seed, unsigned drop_stream, float in_scale, unsigned in_thresh16,
            unsigned in_stream, const unsigned long long* __restrict__ drop_offset = nullptr) {
    extern __shared__ float4 sm4[];  // [gamma: 2*chunks] [warp][3 arrays][2 halves][chunks]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunks = H >> 3;
    float4* sgam = sm4;
    float4* acc = sm4 + 2 * chunks + warp * 6 * chunks;
    pdl_trigger();
    if constexpr (SUMS)
        for (int i = threadIdx.x; i < kLnWarps * 6 * chunks; i += blockDim.x) sm4[2 * chunks + i] = make_float4(0.f, 0.f, 0.f, 0.f);
    pdl_wait();  // the accumulators are cleared while the previous kernel drains; global memory is touched from here on
    // OFF: the hash keys of the summed seed wait in shared memory (the 64-bit sum held in registers spills the NC = 4 build)
    __shared__ uint32_t s_key[2];   // [0]: hidden dropout (drop_stream), [1]: in_dropout (in_stream)
    if constexpr (OFF) {
        if (threadIdx.x == 0) {
            const unsigned long long sd = drop_seed + *drop_offset;
            s_key[0] = dropout_key(sd, drop_stream);
            s_key[1] = dropout_key(sd, in_stream);
        }
    }
    for (int i = threadIdx.x; i < 2 * chunks; i += blockDim.x) {
        const int h = i / chunks, ch = i % chunks;
        sgam[i] = __ldg(reinterpret_cast<const float4*>(gamma + ch * 8 + h * 4));
    }
    __syncthreads();

    const float invH = 1.0f / H;
    // The packed row (ux, ud) is dead once it is unpacked to fp32: the NEXT row of this warp is requested right there, so its
    // 3 KB travel under the two passes over the current row (before: loads and arithmetic alternated, ~48 KB in flight per SM).
    const int rstride = gridDim.x * kLnWarps;
    int row = blockIdx.x * kLnWarps + warp;
    uint4 ux[NC], ud[NC];
    float mu = 0.f, rs = 0.f;
    auto request = [&](int rw) {
        const long long rb = static_cast<long long>(rw) * H;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int ch = lane + c * 32;
            if (ch < chunks) {
                ux[c] = ldg_v4(x + rb + ch * 8);
                ud[c] = ldg_v4(dy + rb + ch * 8);
            }
        }
        mu = mean[rw];
        rs = rstd[rw];
    };
    if (row < rows) request(row);
    for (; row < rows; row += rstride) {
        const long long rbase = static_cast<long long>(row) * H;
        const unsigned long long e8row = static_cast<unsigned long long>(row) * static_cast<unsigned>(chunks);
        const float nmr = -mu * rs;
        const float rs_cur = rs;
        // the row is unpacked ONCE: xh = xhat and dv = dy stay in fp32 registers for both passes (the kernel is
        // instruction-issue bound, not register/occupancy bound)
        float xh[NC][8], dv[NC][8];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int ch = lane + c * 32;
            if (ch < chunks) {
                unpack8(ux[c], xh[c]);
                unpack8(ud[c], dv[c]);
            }
        }
        if (row + rstride < rows) request(row + rstride);
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int ch = lane + c * 32;
            if (ch < chunks) {
                if (in_scale != 0.f) {  // dy is the gradient of dropout(LN(x)): re-apply the keep mask
                    const uint32_t keep = OFF ? dropout_keep8_key(s_key[1], e8row + ch, in_thresh16)
                                              : dropout_keep8(drop_seed, in_stream, e8row + ch, in_thresh16);
#pragma unroll
                    for (int i = 0; i < 8; ++i) dv[c][i] = ((keep >> i) & 1u) ? dv[c][i] * in_scale : 0.f;
                }
                const float4 g0 = sgam[ch], g1 = sgam[chunks + ch];
                const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    xh[c][i] = fmaf(xh[c][i], rs_cur, nmr);  // xhat
                    const float g = dv[c][i] * gm[i];
                    s1 += g;
                    s2 = fmaf(g, xh[c][i], s2);
                }
            }
        }
        const float c1 = warp_sum(s1) * invH, c2 = warp_sum(s2) * invH;
        const float rc1 = rs_cur * c1, rc2 = rs_cur * c2;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int ch = lane + c * 32;
            if (ch < chunks) {
                const float4 g0 = sgam[ch], g1 = sgam[chunks + ch];
                const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
                float o[8];
#pragma unroll
                for (int i = 0; i < 8; ++i)  // rs * (g - c1 - xhat * c2)
                    o[i] = fmaf(-xh[c][i], rc2, fmaf(dv[c][i] * gm[i], rs_cur, -rc1));
                stg_v4(dx + rbase + ch * 8, pack8(o));
                if (dx_drop != nullptr) {
                    const uint32_t keep = OFF ? dropout_keep8_key(s_key[0], e8row + ch, drop_thresh16)
                                              : dropout_keep8(drop_seed, drop_stream, e8row + ch, drop_thresh16);
#pragma unroll
                    for (int i = 0; i < 8; ++i) o[i] = ((keep >> i) & 1u) ? o[i] * drop_scale : 0.f;
                    stg_v4(dx_drop + rbase + ch * 8, pack8(o));
                }
                if constexpr (SUMS) {
                    const float* d = dv[c];
                    const float* h = xh[c];
                    float4 a;
                    a = acc[slot(0, 0, ch, chunks)]; a.x = fmaf(d[0], h[0], a.x); a.y = fmaf(d[1], h[1], a.y); a.z = fmaf(d[2], h[2], a.z); a.w = fmaf(d[3], h[3], a.w); acc[slot(0, 0, ch, chunks)] = a;
                    a = acc[slot(0, 1, ch, chunks)]; a.x = fmaf(d[4], h[4], a.x); a.y = fmaf(d[5], h[5], a.y); a.z = fmaf(d[6], h[6], a.z); a.w = fmaf(d[7], h[7], a.w); acc[slot(0, 1, ch, chunks)] = a;
                    a = acc[slot(1, 0, ch, chunks)]; a.x += d[0]; a.y += d[1]; a.z += d[2]; a.w += d[3]; acc[slot(1, 0, ch, chunks)] = a;
                    a = acc[slot(1, 1, ch, chunks)]; a.x += d[4]; a.y += d[5]; a.z += d[6]; a.w += d[7]; acc[slot(1, 1, ch, chunks)] = a;
                    a = acc[slot(2, 0, ch, chunks)]; a.x += o[0]; a.y += o[1]; a.z += o[2]; a.w += o[3]; acc[slot(2, 0, ch, chunks)] = a;
                    a = acc[slot(2, 1, ch, chunks)]; a.x += o[4]; a.y += o[5]; a.z += o[6]; a.w += o[7]; acc[slot(2, 1, ch, chunks)] = a;
                }
            }
        }
    }
    if constexpr (!SUMS) return;
    __syncthreads();
    // reduce the 8 warp slabs and flush: one global atomic per column per array per block
    const float* accf = reinterpret_cast<const float*>(sm4 + 2 * chunks);
    for (int i = threadIdx.x; i < 3 * H; i += blockDim.x) {
        const int a = i / H, col = i % H;
        const int ch = col >> 3, h = (col >> 2) & 1, e = col & 3;
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < kLnWarps; ++w) s += accf[(w * 6 * chunks + slot(a, h, ch, chunks)) * 4 + e];
        if constexpr (PART) {
            dgamma[static_cast<long long>(blockIdx.x) * 3 * H + i] = s;
        } else {
            float* dst = a == 0 ? dgamma : (a == 1 ? dbeta : dbias);
            if (dst != nullptr) atomicAdd(dst + col, s);
        }
    }
}

#define VB_LN_BWD_PARAMS                                                                                                       \
    const bf16 *__restrict__ dy, const bf16 *__restrict__ x, const float *__restrict__ mean, const float *__restrict__ rstd,   \
        const float *__restrict__ gamma, bf16 *__restrict__ dx, bf16 *__restrict__ dx_drop, float *__restrict__ dgamma,        \
        float *__restrict__ dbeta, float *__restrict__ dbias, int rows, int H, float drop_scale, unsigned drop_thresh16,      \
        unsigned long long drop_seed, unsigned drop_stream, float in_scale, unsigned in_thresh16, unsigned in_stream
#define VB_LN_BWD_ARGS \
    dy, x, mean, rstd, gamma, dx, dx_drop, dgamma, dbeta, dbias, rows, H, drop_scale, drop_thresh16, drop_seed, drop_stream, in_scale, in_thresh16, in_stream
template <int NC>
__global__ void __launch_bounds__(kLnWarps * 32, 2) ln_bwd_kernel(VB_LN_BWD_PARAMS) { ln_bwd_body<NC, false>(VB_LN_BWD_ARGS); }
template <int NC>
__global__ void __launch_bounds__(kLnWarps * 32, 2) ln_bwd_part_kernel(VB_LN_BWD_PARAMS) { ln_bwd_body<NC, true>(VB_LN_BWD_ARGS); }
template <int NC>
__global__ void __launch_bounds__(kLnWarps * 32, 2)
ln_bwd_off_kernel(VB_LN_BWD_PARAMS, const unsigned long long* __restrict__ drop_offset) {
    ln_bwd_body<NC, false, true>(VB_LN_BWD_ARGS, drop_offset);
}
template <int NC>
__global__ void __launch_bounds__(kLnWarps * 32, 2)
ln_bwd_part_off_kernel(VB_LN_BWD_PARAMS, const unsigned long long* __restrict__ drop_offset) {
    ln_bwd_body<NC, true, true>(VB_LN_BWD_ARGS, drop_offset);
}
template <int NC>
__global__ void __launch_bounds__(kLnWarps * 32, 2)
ln_bwd_rows_kernel(VB_LN_BWD_PARAMS) { ln_bwd_body<NC, false, false, false>(VB_LN_BWD_ARGS); }
// NC = 4 with the offset spills at 2 blocks per SM (128 registers): one block per SM there, two everywhere else
template <int NC>
__global__ void __launch_bounds__(kLnWarps * 32, NC == 4 ? 1 : 2)
ln_bwd_rows_off_kernel(VB_LN_BWD_PARAMS, const unsigned long long* __restrict__ drop_offset) {
    ln_bwd_body<NC, false, true, false>(VB_LN_BWD_ARGS, drop_offset);
}
#undef VB_LN_BWD_PARAMS
#undef VB_LN_BWD_ARGS

// out_j[i % seg] += sum_p part[p * width + i] for i in [0, width), j = i / seg (null outputs are skipped): the block partials of a
// deterministic-mode column reduction, added in partial order. One thread per column; consecutive threads read consecutive columns.
__global__ void __launch_bounds__(256)
partials_reduce_kernel(const float* __restrict__ part, int parts, int width, int seg, float* o0, float* o1, float* o2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= width) return;
    float s = 0.f;
    for (int p = 0; p < parts; ++p) s += part[static_cast<long long>(p) * width + i];
    const int j = i / seg;
    float* o = j == 0 ? o0 : (j == 1 ? o1 : o2);
    if (o != nullptr) o[i - j * seg] += s;
}

int partials_reduce(const float* part, int parts, int width, int seg, float* o0, float* o1, float* o2, cudaStream_t st) {
    {
        ProfScope ps(st, PROF_COLSUM, 4.0 * parts * width, 1);
        partials_reduce_kernel<<<(width + 255) / 256, 256, 0, st>>>(part, parts, width, seg, o0, o1, o2);
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// grid of ln_bwd: 2 resident blocks per SM (123 registers: the row is cached in fp32; an 80-register / 3-block build spills and
// measured 30 % slower), fewer when there are fewer row groups
static int ln_bwd_grid(int rows) {
    int grid = num_sms() * 2;
    const int need = (rows + kLnWarps - 1) / kLnWarps;
    return grid > need ? need : grid;
}
long long ln_bwd_det_bytes(int rows, int H) { return static_cast<long long>(ln_bwd_grid(rows)) * 3 * H * 4; }

int ln_fwd(const void* x, long long ldx, const float* gamma, const float* beta, void* y, long long ldy,
           float* mean, float* rstd, int rows, int H, float eps, cudaStream_t st) {
    VB_REQUIRE(H % 8 == 0 && H <= 1024 * 2, "layernorm: H=%d must be a multiple of 8 and <= 2048", H);
    VB_REQUIRE(rows > 0, "layernorm: no rows");
    VB_REQUIRE(x && y && gamma && beta, "layernorm: x, y, gamma and beta must not be NULL");
    VB_REQUIRE(ldx >= H && ldy >= H && ldx % 8 == 0 && ldy % 8 == 0,
               "layernorm: ldx=%lld and ldy=%lld must be multiples of 8 and >= H=%d", ldx, ldy, H);
    VB_REQUIRE(all_aligned16(x, y, gamma, beta), "layernorm: x, y, gamma and beta must be 16-byte aligned");
    const int nc = (H / 8 + 31) / 32;
    const int grid = (rows + kLnWarps - 1) / kLnWarps;
    const bf16* xb = static_cast<const bf16*>(x);
    bf16* yb = static_cast<bf16*>(y);
    ProfScope ps(st, PROF_LN_FWD, 4.0 * rows * H, 1);  // bytes: read + write bf16
#define VB_LN_FWD(NC) \
    VB_CHECK_CUDA(launch_pdl(ln_fwd_kernel<NC>, dim3(grid), dim3(kLnWarps * 32), 0, st, xb, ldx, gamma, beta, yb, ldy, mean, rstd, rows, H, eps))
    switch (nc) {
        case 1: VB_LN_FWD(1); break;
        case 2: VB_LN_FWD(2); break;
        case 3: VB_LN_FWD(3); break;
        case 4: VB_LN_FWD(4); break;
        default: VB_LN_FWD(8); break;
    }
#undef VB_LN_FWD
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int ln_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const float* gamma, void* dx,
           void* dx_drop, float* dgamma, float* dbeta, float* dbias, int rows, int H, float dropout_p,
           unsigned long long seed, unsigned stream_id, float in_dropout_p, unsigned in_stream_id, cudaStream_t st,
           bool rows_only) {
    VB_REQUIRE(H % 8 == 0 && H <= 1024, "layernorm backward: H=%d must be a multiple of 8 and <= 1024", H);
    VB_REQUIRE(rows > 0, "layernorm backward: no rows");
    VB_REQUIRE((dropout_p > 0.f) == (dx_drop != nullptr), "layernorm backward: dx_drop iff dropout_p > 0");
    VB_REQUIRE(dy && x && mean && rstd && gamma && dx, "layernorm backward: dy, x, mean, rstd, gamma and dx must not be NULL");
    VB_REQUIRE(all_aligned16(dy, x, gamma, dx, dx_drop), "layernorm backward: dy, x, gamma, dx and dx_drop must be 16-byte aligned");
    const int nc = (H / 8 + 31) / 32;
    const int grid = ln_bwd_grid(rows);
    VB_REQUIRE(!rows_only || (!dgamma && !dbeta && !dbias), "layernorm backward: a row-only call takes no column sums");
    const DetWs det = det_ws();
    if (det.ptr != nullptr && !rows_only) VB_TRY_RC(det_require(ln_bwd_det_bytes(rows, H), "layernorm backward"));
    // the offset kernels only when this call draws dropout bits (hidden dropout or the embeddings' in_dropout)
    const unsigned long long* off = (dropout_p > 0.f || in_dropout_p > 0.f) ? drop_offset() : nullptr;
    const DropQ dq = dropout_quantise(dropout_p), iq = dropout_quantise(in_dropout_p);
    const float scale = dq.scale, in_scale = iq.scale;
    const unsigned th = dq.thr8, in_th = iq.thr8;
    if (rows_only) {   // same arithmetic per row, no column reductions: deterministic mode has nothing to order
        const size_t rsmem = static_cast<size_t>(2 * (H / 8)) * sizeof(float4);
        {
            ProfScope ps(st, PROF_LN_BWD, (dx_drop ? 8.0 : 6.0) * rows * H, 1);
#define VB_LN_ROWS(K, NC, ...)                                                                               \
    VB_CHECK_CUDA(launch_pdl(K<NC>, dim3(grid), dim3(kLnWarps * 32), rsmem, st,                             \
        static_cast<const bf16*>(dy), static_cast<const bf16*>(x), mean, rstd, gamma, static_cast<bf16*>(dx), \
        static_cast<bf16*>(dx_drop), nullptr, nullptr, nullptr, rows, H, scale, th, seed, stream_id,          \
        in_scale, in_th, __VA_ARGS__))
            if (off != nullptr) {
                switch (nc) {
                    case 1: VB_LN_ROWS(ln_bwd_rows_off_kernel, 1, in_stream_id, off); break;
                    case 2: VB_LN_ROWS(ln_bwd_rows_off_kernel, 2, in_stream_id, off); break;
                    case 3: VB_LN_ROWS(ln_bwd_rows_off_kernel, 3, in_stream_id, off); break;
                    default: VB_LN_ROWS(ln_bwd_rows_off_kernel, 4, in_stream_id, off); break;
                }
            } else {
                switch (nc) {
                    case 1: VB_LN_ROWS(ln_bwd_rows_kernel, 1, in_stream_id); break;
                    case 2: VB_LN_ROWS(ln_bwd_rows_kernel, 2, in_stream_id); break;
                    case 3: VB_LN_ROWS(ln_bwd_rows_kernel, 3, in_stream_id); break;
                    default: VB_LN_ROWS(ln_bwd_rows_kernel, 4, in_stream_id); break;
                }
            }
#undef VB_LN_ROWS
        }
        VB_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    const size_t smem = static_cast<size_t>(2 * (H / 8) + kLnWarps * 6 * (H / 8)) * sizeof(float4);
    static int cfg1[kMaxDevices] = {0}, cfg2[kMaxDevices] = {0}, cfg3[kMaxDevices] = {0}, cfg4[kMaxDevices] = {0};
    VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_kernel<1>, 100 * 1024, cfg1));
    VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_kernel<2>, 100 * 1024, cfg2));
    VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_kernel<3>, 100 * 1024, cfg3));
    VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_kernel<4>, 100 * 1024, cfg4));
    if (off != nullptr) {
        static int ocfg[2][4][kMaxDevices] = {};
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_off_kernel<1>, 100 * 1024, ocfg[0][0]));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_off_kernel<2>, 100 * 1024, ocfg[0][1]));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_off_kernel<3>, 100 * 1024, ocfg[0][2]));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_off_kernel<4>, 100 * 1024, ocfg[0][3]));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_part_off_kernel<1>, 100 * 1024, ocfg[1][0]));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_part_off_kernel<2>, 100 * 1024, ocfg[1][1]));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_part_off_kernel<3>, 100 * 1024, ocfg[1][2]));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_part_off_kernel<4>, 100 * 1024, ocfg[1][3]));
    }
    if (det.ptr != nullptr) {
        static int dcfg1[kMaxDevices] = {0}, dcfg2[kMaxDevices] = {0}, dcfg3[kMaxDevices] = {0}, dcfg4[kMaxDevices] = {0};
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_part_kernel<1>, 100 * 1024, dcfg1));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_part_kernel<2>, 100 * 1024, dcfg2));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_part_kernel<3>, 100 * 1024, dcfg3));
        VB_CHECK_CUDA(ensure_dyn_smem(ln_bwd_part_kernel<4>, 100 * 1024, dcfg4));
    }
    {
        ProfScope ps(st, PROF_LN_BWD, (dx_drop ? 8.0 : 6.0) * rows * H, 1);
#define VB_LN_BWD(K, NC, DG)                                                                                 \
    VB_CHECK_CUDA(launch_pdl(K<NC>, dim3(grid), dim3(kLnWarps * 32), smem, st,                              \
        static_cast<const bf16*>(dy), static_cast<const bf16*>(x), mean, rstd, gamma, static_cast<bf16*>(dx), \
        static_cast<bf16*>(dx_drop), DG, dbeta, dbias, rows, H, scale, th, seed, stream_id, in_scale,        \
        in_th, in_stream_id))
#define VB_LN_BWD_OFF(K, NC, DG)                                                                             \
    VB_CHECK_CUDA(launch_pdl(K<NC>, dim3(grid), dim3(kLnWarps * 32), smem, st,                              \
        static_cast<const bf16*>(dy), static_cast<const bf16*>(x), mean, rstd, gamma, static_cast<bf16*>(dx), \
        static_cast<bf16*>(dx_drop), DG, dbeta, dbias, rows, H, scale, th, seed, stream_id, in_scale,        \
        in_th, in_stream_id, off))
        if (off != nullptr) {
            float* part = static_cast<float*>(det.ptr);
            if (det.ptr != nullptr) {
                switch (nc) {
                    case 1: VB_LN_BWD_OFF(ln_bwd_part_off_kernel, 1, part); break;
                    case 2: VB_LN_BWD_OFF(ln_bwd_part_off_kernel, 2, part); break;
                    case 3: VB_LN_BWD_OFF(ln_bwd_part_off_kernel, 3, part); break;
                    default: VB_LN_BWD_OFF(ln_bwd_part_off_kernel, 4, part); break;
                }
            } else {
                switch (nc) {
                    case 1: VB_LN_BWD_OFF(ln_bwd_off_kernel, 1, dgamma); break;
                    case 2: VB_LN_BWD_OFF(ln_bwd_off_kernel, 2, dgamma); break;
                    case 3: VB_LN_BWD_OFF(ln_bwd_off_kernel, 3, dgamma); break;
                    default: VB_LN_BWD_OFF(ln_bwd_off_kernel, 4, dgamma); break;
                }
            }
        } else if (det.ptr != nullptr) {
            float* part = static_cast<float*>(det.ptr);
            switch (nc) {
                case 1: VB_LN_BWD(ln_bwd_part_kernel, 1, part); break;
                case 2: VB_LN_BWD(ln_bwd_part_kernel, 2, part); break;
                case 3: VB_LN_BWD(ln_bwd_part_kernel, 3, part); break;
                default: VB_LN_BWD(ln_bwd_part_kernel, 4, part); break;
            }
        } else {
            switch (nc) {
                case 1: VB_LN_BWD(ln_bwd_kernel, 1, dgamma); break;
                case 2: VB_LN_BWD(ln_bwd_kernel, 2, dgamma); break;
                case 3: VB_LN_BWD(ln_bwd_kernel, 3, dgamma); break;
                default: VB_LN_BWD(ln_bwd_kernel, 4, dgamma); break;
            }
        }
#undef VB_LN_BWD
#undef VB_LN_BWD_OFF
    }
    VB_CHECK_CUDA(cudaGetLastError());
    if (det.ptr != nullptr) return partials_reduce(static_cast<const float*>(det.ptr), grid, 3 * H, H, dgamma, dbeta, dbias, st);
    return 0;
}

}  // namespace vb

extern "C" {
int vb_layernorm_fwd(const void* x, int64_t ldx, const float* gamma, const float* beta, void* y, int64_t ldy,
                     float* mean, float* rstd, int32_t rows, int32_t hidden, float eps, void* stream) {
    return vb::ln_fwd(x, ldx, gamma, beta, y, ldy, mean, rstd, rows, hidden, eps, static_cast<cudaStream_t>(stream));
}
int vb_layernorm_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const float* gamma,
                     void* dx, void* dx_drop, float* dgamma, float* dbeta, float* dbias, int32_t rows,
                     int32_t hidden, float dropout_p, uint64_t dropout_seed, uint32_t dropout_stream,
                     float in_dropout_p, uint32_t in_dropout_stream, void* stream) {
    return vb::ln_bwd(dy, x, mean, rstd, gamma, dx, dx_drop, dgamma, dbeta, dbias, rows, hidden, dropout_p,
                      dropout_seed, dropout_stream, in_dropout_p, in_dropout_stream, static_cast<cudaStream_t>(stream), false);
}
}
