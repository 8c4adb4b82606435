// vb_attention_head.cu — persistent whole-head mma.sync attention kernels for 192 < seq <= 256 (beyond the wgmma kernels
// of vb_attention_wgmma.cu, whose backward does not fit in shared memory there).
//
// The staged kernels in vb_attention.cu launch one short-lived CTA per (batch, head, 64-query block): each
// re-loads the head's K/V and spends much of its short life waiting for that load. Here one CTA owns a whole (batch, head): NW = 16 warps, each with 16 query rows
// (and, in backward, 16 key rows); Q/K/V (and dO) tiles are loaded ONCE per head with cp.async, and the CTA is
// persistent — it walks over heads and prefetches the next head's tiles into the second shared-memory buffer
// while computing the current one, so the tensor pipe never waits for HBM/L2 latency.
//
//   forward   smem 2 x (Q, K, V) tiles          S=256: 2 x 96 KB   16 warps/CTA, 1 CTA/SM
//   backward  delta pre-kernel: D = rowsum(dO * O)  (HBM-bound, one warp per token)
//             fused kernel: smem (Q, K, V, dO) x {1,2} buffers; phase A: dQ (rows = queries),
//             phase B: dK, dV (rows = keys) — the tiles are shared by both phases (loaded once, not 2 x 3 times).
#include "vb_attention.cuh"

namespace vb {

// ------------------------------------------------------------------------------------------------
// tile loading: nkb 64-row tiles of one head slice, all threads of the CTA
// ------------------------------------------------------------------------------------------------
template <int NT>
__device__ __forceinline__ void load_rows(uint32_t tiles, const bf16* base, long long ld, int nkb, int S, int tid) {
    for (int idx = tid; idx < nkb * 512; idx += NT) {  // 512 16-byte chunks per 64x64 tile
        const int tile = idx >> 9, r = (idx >> 3) & 63, c = idx & 7;
        const int row = tile * kBlk + r;
        const bool ok = row < S;
        cp_async16(tiles + tile * kTileBytes + swz(r, c), base + static_cast<long long>(ok ? row : 0) * ld + c * 8, ok);
    }
}

// ------------------------------------------------------------------------------------------------
// attention-probability dropout mask: one thread per 64-bit word (query row, 64-key block), 16 counter hashes -> 64 keep
// decisions of 8 random bits each (keep iff value >= thresh8). Drawing the bits inside the attention kernels made them
// slower than this separate pass, which has nothing else to do and runs at full issue rate.
// Two layouts are written: keep[(bh * np64 + q) * nkb + kb] (bit = key % 64; rows = queries: forward kernels, mma.sync
// backward) and the transpose keepT[(bh * np64 + key) * nkb + qb] (bit = query % 64; rows = keys: for a backward
// that walks keys). A block is one 64 x 64 bit tile; the transpose is 64 warp ballots per 32 rows.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void
attn_keep_mask_body(unsigned long long* __restrict__ keep, unsigned long long* __restrict__ keepT, int nkb, int np64, int S,
                    unsigned seed, unsigned thresh8) {
    const int kb = blockIdx.x % nkb, qb = (blockIdx.x / nkb) % nkb;
    const long long bh = blockIdx.x / (nkb * nkb);
    const int row = qb * 64 + threadIdx.x;
    const long long w = (bh * np64 + row) * nkb + kb;
    unsigned long long word = ~0ull;
    if (row < S) {
        // bit-sliced comparison: 8 hashes are the 8 bit-planes of 32 independent 8-bit random values v; keep iff v >= thresh8
        // (MSB-first comparator: ~2 logic ops per plane for 32 decisions, instead of a byte-wise compare per hash)
        const uint32_t base = static_cast<uint32_t>(w) * 16u;
        uint32_t half_w[2];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            uint32_t ge = 0u, eq = 0xffffffffu;
#pragma unroll
            for (int b = 7; b >= 0; --b) {
                const uint32_t plane = mix32((base + half * 8 + b) ^ seed);
                const uint32_t tb = 0u - ((thresh8 >> b) & 1u);  // all ones when the threshold bit is set
                ge |= eq & plane & ~tb;                            // threshold bit 0, value bit 1: greater
                eq &= ~(plane ^ tb);                               // still equal on this bit
            }
            half_w[half] = ge | eq;
        }
        word = static_cast<unsigned long long>(half_w[0]) | (static_cast<unsigned long long>(half_w[1]) << 32);
    }
    keep[w] = word;
    // transpose the warp's two 32 x 32 bit blocks (rows = this warp's queries, columns = keys 0-31 / 32-63 of the block)
    // with a 5-round shuffle butterfly: afterwards lane l holds, for key l (resp. 32 + l), the bits of the warp's 32 queries
    const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
    uint32_t t_lo = static_cast<uint32_t>(word), t_hi = static_cast<uint32_t>(word >> 32);
#pragma unroll
    for (int j = 16; j >= 1; j >>= 1) {
        const uint32_t m0 = j == 16 ? 0x0000ffffu : j == 8 ? 0x00ff00ffu : j == 4 ? 0x0f0f0f0fu : j == 2 ? 0x33333333u : 0x55555555u;
        const uint32_t y_lo = __shfl_xor_sync(0xffffffffu, t_lo, j), y_hi = __shfl_xor_sync(0xffffffffu, t_hi, j);
        if ((lane & j) == 0) {
            t_lo = (t_lo & m0) | ((y_lo & m0) << j);
            t_hi = (t_hi & m0) | ((y_hi & m0) << j);
        } else {
            t_lo = ((y_lo & ~m0) >> j) | (t_lo & ~m0);
            t_hi = ((y_hi & ~m0) >> j) | (t_hi & ~m0);
        }
    }
    uint32_t* kt32 = reinterpret_cast<uint32_t*>(keepT);
    kt32[((bh * np64 + kb * 64 + lane) * nkb + qb) * 2 + wi] = t_lo;
    kt32[((bh * np64 + kb * 64 + 32 + lane) * nkb + qb) * 2 + wi] = t_hi;
}
__global__ void __launch_bounds__(64)
attn_keep_mask_kernel(unsigned long long* __restrict__ keep, unsigned long long* __restrict__ keepT, int nkb, int np64, int S,
                      unsigned seed, unsigned thresh8) {
    pdl_trigger();
    pdl_wait();
    attn_keep_mask_body(keep, keepT, nkb, np64, S, seed, thresh8);
}
// vb_set_dropout_offset: the seed is folded from seed64 + *offset, read once the previous kernel's writes are visible
__global__ void __launch_bounds__(64)
attn_keep_mask_off_kernel(unsigned long long* __restrict__ keep, unsigned long long* __restrict__ keepT, int nkb, int np64, int S,
                          unsigned long long seed64, unsigned stream_id, const unsigned long long* __restrict__ offset, unsigned thresh8) {
    pdl_trigger();
    pdl_wait();
    attn_keep_mask_body(keep, keepT, nkb, np64, S, attn_seed_fold(seed64 + *offset, stream_id), thresh8);
}

// one 64-key block of the forward pass for a 16-row warp tile (same math as the staged kernel)
__device__ __forceinline__ void fwd_block(const AttnParams& p, float (&o)[8][4], float (&m)[2], float (&l)[2],
                                          const uint32_t (&qf)[4][4], uint32_t sK, uint32_t sV, const float* sbias,
                                          int kb, int kvalid, int qrow0, unsigned bh, int nkb, int lane, float sc2) {
    const int g = lane >> 2, t = lane & 3;
    // keep bits of the two query rows of this lane for this key block (written by attn_keep_mask_kernel): issued before
    // the QK^T MMAs so the loads are back long before the bits are needed
    unsigned long long keep_a = ~0ull, keep_c = ~0ull;
    if (p.drop_scale != 0.f) {
        const unsigned long long* kp = p.keep + (static_cast<unsigned long long>(bh) * (nkb * kBlk)) * nkb;
        keep_a = kp[static_cast<long long>(qrow0 + g) * nkb + kb];
        keep_c = kp[static_cast<long long>(qrow0 + g + 8) * nkb + kb];
    }
    float s[8][4];
    zero_acc(s);
    gemm_nt(s, qf, sK, lane, kvalid);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        const float b0 = sbias[nt * 8 + 2 * t], b1 = sbias[nt * 8 + 2 * t + 1];
        s[nt][0] = fmaf(s[nt][0], sc2, b0); s[nt][1] = fmaf(s[nt][1], sc2, b1);
        s[nt][2] = fmaf(s[nt][2], sc2, b0); s[nt][3] = fmaf(s[nt][3], sc2, b1);
        mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
        mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float mn = fmaxf(m[r], mx[r]);
        alpha[r] = fast_ex2(m[r] - mn);
        m[r] = mn;
    }
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        s[nt][0] = fast_ex2(s[nt][0] - m[0]); s[nt][1] = fast_ex2(s[nt][1] - m[0]);
        s[nt][2] = fast_ex2(s[nt][2] - m[1]); s[nt][3] = fast_ex2(s[nt][3] - m[1]);
        rs[0] += s[nt][0] + s[nt][1];
        rs[1] += s[nt][2] + s[nt][3];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
        rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
        l[r] = l[r] * alpha[r] + rs[r];
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        o[nt][0] *= alpha[0]; o[nt][1] *= alpha[0];
        o[nt][2] *= alpha[1]; o[nt][3] *= alpha[1];
    }
    if (p.drop_scale != 0.f) {
        // the lane's bits sit at 8*nt + 2*t + {0, 1}: shift by 2*t once, then every test is at a compile-time position.
        // The 1/(1-p) factor is NOT applied here: it is folded into the final 1/l normalisation of the output row.
        const uint32_t alo = static_cast<uint32_t>(keep_a >> (2 * t)), ahi = static_cast<uint32_t>(keep_a >> (2 * t + 32));
        const uint32_t clo = static_cast<uint32_t>(keep_c >> (2 * t)), chi = static_cast<uint32_t>(keep_c >> (2 * t + 32));
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const uint32_t wa = nt < 4 ? alo : ahi, wc = nt < 4 ? clo : chi;
            const int sh = 8 * (nt & 3);
            s[nt][0] = ((wa >> sh) & 1u) ? s[nt][0] : 0.f;
            s[nt][1] = ((wa >> (sh + 1)) & 1u) ? s[nt][1] : 0.f;
            s[nt][2] = ((wc >> sh) & 1u) ? s[nt][2] : 0.f;
            s[nt][3] = ((wc >> (sh + 1)) & 1u) ? s[nt][3] : 0.f;
        }
    }
    uint32_t pf[4][4];
    acc_to_afrag(pf, s);
    gemm_nn(o, pf, sV, lane, kvalid);
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
template <int NW, bool VL = false>
__global__ void __launch_bounds__(NW * 32, 1)
attn_fwd_head_kernel(const AttnParams p, const int nkb) {
    constexpr int NT = NW * 32;
    extern __shared__ __align__(128) uint8_t dsmem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int S = p.S;
    const long long ld = 3LL * p.H;
    const int buf_bytes = 3 * nkb * kTileBytes;
    float* sbias_all = reinterpret_cast<float*>(dsmem + 2 * buf_bytes);  // [2][nkb*64]
    const int total = p.B * p.A;
    const float sc2 = p.scale * kLog2e;
    const int qrow0 = warp * 16;
    const bool active = qrow0 < S;

    auto issue = [&](int item, int buf) {
        const int b = item / p.A, h = item % p.A;
        const SeqSpan sp = seq_span<VL>(p, b, h);
        const int nkv = VL ? (sp.len + kBlk - 1) / kBlk : nkb;  // tiles past the sequence's end are not loaded
        const bf16* qbase = p.qkv + sp.row0 * ld + h * kHd;
        const uint32_t base = smem_u32(dsmem) + buf * buf_bytes;
        load_rows<NT>(base, qbase, ld, nkv, sp.len, tid);
        load_rows<NT>(base + nkb * kTileBytes, qbase + p.H, ld, nkv, sp.len, tid);
        load_rows<NT>(base + 2 * nkb * kTileBytes, qbase + 2 * p.H, ld, nkv, sp.len, tid);
        cp_async_commit();
        float* sb = sbias_all + buf * nkb * kBlk;
        for (int i = tid; i < nkb * kBlk; i += NT) sb[i] = key_bias2<VL>(p, b, i, sp.len);
    };

    int item = blockIdx.x;
    if (item >= total) return;
    pdl_trigger();
    pdl_wait();
    issue(item, 0);
    int buf = 0;
    for (; item < total; item += gridDim.x, buf ^= 1) {
        const int next = item + gridDim.x;
        if (next < total) {
            issue(next, buf ^ 1);  // prefetch the next head while this one is computed
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const int b = item / p.A, h = item % p.A;
        const SeqSpan sp = seq_span<VL>(p, b, h);
        const int len = sp.len;
        if (VL ? qrow0 < len : active) {  // warps past the sequence's end skip the head
            const unsigned bh = static_cast<unsigned>(item);
            const uint32_t base = smem_u32(dsmem) + buf * buf_bytes;
            const float* sb = sbias_all + buf * nkb * kBlk;
            const int nkv = VL ? (len + kBlk - 1) / kBlk : nkb;
            uint32_t qf[4][4];
            load_afrag(qf, base + (warp >> 2) * kTileBytes, (warp & 3) * 16, lane);
            float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
            float o[8][4];
            zero_acc(o);
            for (int kb = 0; kb < nkv; ++kb) {
                const int kvalid = min(kBlk, len - kb * kBlk);
                fwd_block(p, o, m, l, qf, base + (nkb + kb) * kTileBytes, base + (2 * nkb + kb) * kTileBytes,
                          sb + kb * kBlk, kb, kvalid, qrow0, bh, nkb, lane, sc2);
            }
            const float dscale = p.drop_scale != 0.f ? p.drop_scale : 1.f;  // survivors' 1/(1-p), see fwd_block
            const float inv0 = dscale / l[0], inv1 = dscale / l[1];
            store_acc(p.ctx + sp.row0 * p.H + h * kHd, p.H, qrow0, len, o, lane, inv0, inv1);
            if (t == 0 && p.lse != nullptr) {
                float* lse = p.lse + (VL ? sp.stat0 : static_cast<long long>(item) * S);
                if (qrow0 + g < len) lse[qrow0 + g] = (m[0] + log2f(l[0])) * 0.6931471805599453f;
                if (qrow0 + g + 8 < len) lse[qrow0 + g + 8] = (m[1] + log2f(l[1])) * 0.6931471805599453f;
            }
        }
        __syncthreads();  // buffer `buf` is free again: the prefetch two iterations ahead may overwrite it
    }
}

// ------------------------------------------------------------------------------------------------
// backward: delta pre-kernel  D[b, h, q] = sum_d dO[b, q, h, d] * O[b, q, h, d]
// ------------------------------------------------------------------------------------------------
// VL (variable-length calls): rows are the `total` packed tokens and drow is [A, total] (B = 1, S = total below)
template <bool VL = false>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ d_o, float* __restrict__ drow, int B, int S,
                  int A, int H) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = static_cast<long long>(blockIdx.x) * 8 + warp;  // token index b*S + q
    pdl_trigger();
    pdl_wait();
    if (row >= static_cast<long long>(B) * S) return;
    const int b = VL ? 0 : static_cast<int>(row / S), q = VL ? static_cast<int>(row) : static_cast<int>(row % S);
    const int chunks = H >> 3;  // 8 chunks of 8 elements per head
    for (int c0 = 0; c0 < chunks; c0 += 32) {  // warp-uniform trip count: the shuffles below need all lanes
        const int ch = c0 + lane;
        float s = 0.f;
        if (ch < chunks) {
            const uint4 a = ldg_v4(o + row * H + ch * 8), c = ldg_v4(d_o + row * H + ch * 8);
            const uint32_t av[4] = {a.x, a.y, a.z, a.w}, cv[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 x = unpack_bf16x2(av[i]), y = unpack_bf16x2(cv[i]);
                s += x.x * y.x + x.y * y.y;
            }
        }
        // the 8 lanes holding one head's chunks are contiguous and 8-aligned (32 % 8 == 0)
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        if ((lane & 7) == 0 && ch < chunks) drow[(static_cast<long long>(b) * A + (ch >> 3)) * S + q] = s;
    }
}

// ------------------------------------------------------------------------------------------------
// backward: fused dQ + dK/dV for one (batch, head) per CTA iteration
// smem per buffer: Q | K | V | dO tiles (nkb each) ; then per buffer fp32 arrays lse2[nkb*64], D[nkb*64], bias2[nkb*64]
// ------------------------------------------------------------------------------------------------
template <int NW, bool VL = false>
__global__ void __launch_bounds__(NW * 32, 1)
attn_bwd_head_kernel(const AttnParams p, const int nkb, const int nbuf) {
    constexpr int NT = NW * 32;
    extern __shared__ __align__(128) uint8_t dsmem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int S = p.S;
    const long long ld = 3LL * p.H;
    const int buf_bytes = 4 * nkb * kTileBytes;
    float* svec_all = reinterpret_cast<float*>(dsmem + nbuf * buf_bytes);  // [nbuf][3][nkb*64]
    const int total = p.B * p.A;
    const float sc2 = p.scale * kLog2e;
    const int row0 = warp * 16;
    const bool active = row0 < S;
    const int np64 = nkb * kBlk;

    auto issue = [&](int item, int buf) {
        const int b = item / p.A, h = item % p.A;
        const SeqSpan sp = seq_span<VL>(p, b, h);
        const int len = sp.len, nkv = VL ? (len + kBlk - 1) / kBlk : nkb;
        const bf16* qbase = p.qkv + sp.row0 * ld + h * kHd;
        const bf16* dobase = p.dctx + sp.row0 * p.H + h * kHd;
        const uint32_t base = smem_u32(dsmem) + buf * buf_bytes;
        load_rows<NT>(base, qbase, ld, nkv, len, tid);
        load_rows<NT>(base + nkb * kTileBytes, qbase + p.H, ld, nkv, len, tid);
        load_rows<NT>(base + 2 * nkb * kTileBytes, qbase + 2 * p.H, ld, nkv, len, tid);
        load_rows<NT>(base + 3 * nkb * kTileBytes, dobase, p.H, nkv, len, tid);
        cp_async_commit();
        float* sv = svec_all + buf * 3 * np64;
        const long long stat0 = VL ? sp.stat0 : static_cast<long long>(item) * S;
        const float* lsep = p.lse + stat0;
        const float* drp = p.drow + stat0;
        for (int i = tid; i < np64; i += NT) {
            sv[i] = i < len ? lsep[i] * kLog2e : INFINITY;                       // +inf => p = 0 for padded queries
            sv[np64 + i] = i < len ? drp[i] : 0.f;
            sv[2 * np64 + i] = key_bias2<VL>(p, b, i, len);
        }
    };

    int item = blockIdx.x;
    if (item >= total) return;
    pdl_trigger();
    pdl_wait();
    if (nbuf == 2) issue(item, 0);
    int buf = 0;
    for (; item < total; item += gridDim.x) {
        if (nbuf == 2) {
            const int next = item + gridDim.x;
            if (next < total) { issue(next, buf ^ 1); cp_async_wait<1>(); }
            else cp_async_wait<0>();
        } else {
            issue(item, 0);
            cp_async_wait<0>();
        }
        __syncthreads();
        const int b = item / p.A, h = item % p.A;
        const SeqSpan sp = seq_span<VL>(p, b, h);
        const int len = sp.len, nkv = VL ? (len + kBlk - 1) / kBlk : nkb;
        if (VL ? row0 < len : active) {
            const unsigned bh = static_cast<unsigned>(item);
            const uint32_t base = smem_u32(dsmem) + buf * buf_bytes;
            const uint32_t sQ = base, sK = base + nkb * kTileBytes, sV = base + 2 * nkb * kTileBytes, sdO = base + 3 * nkb * kTileBytes;
            const float* slse = svec_all + buf * 3 * np64;
            const float* sD = slse + np64;
            const float* sbias = slse + 2 * np64;
            const bool drop = p.drop_scale != 0.f;
            const float ds = drop ? p.drop_scale : 1.f;
            bf16* dbase = p.dqkv + sp.row0 * ld + h * kHd;
            const int mytile = warp >> 2, myrow = (warp & 3) * 16;

            // ---------------- phase A: dQ for query rows row0 .. row0+15 ----------------
            {
                uint32_t qf[4][4], dof[4][4];
                load_afrag(qf, sQ + mytile * kTileBytes, myrow, lane);
                load_afrag(dof, sdO + mytile * kTileBytes, myrow, lane);
                const float lse0 = slse[row0 + g], lse1 = slse[row0 + g + 8];
                const float d0 = sD[row0 + g], d1 = sD[row0 + g + 8];
                float dq[8][4];
                zero_acc(dq);
                for (int kb = 0; kb < nkv; ++kb) {
                    const int kvalid = min(kBlk, len - kb * kBlk);
                    unsigned long long keep_a = ~0ull, keep_c = ~0ull;
                    if (drop) {
                        const unsigned long long* kp = p.keep + (static_cast<unsigned long long>(bh) * np64) * nkb;
                        keep_a = kp[static_cast<long long>(row0 + g) * nkb + kb];
                        keep_c = kp[static_cast<long long>(row0 + g + 8) * nkb + kb];
                    }
                    float s[8][4];
                    zero_acc(s);
                    gemm_nt(s, qf, sK + kb * kTileBytes, lane, kvalid);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {  // dP = dO V^T in two 32-key halves (register pressure)
                        float dp[4][4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
                        gemm_nt_half(dp, dof, sV + kb * kTileBytes, lane, hh, kvalid);
#pragma unroll
                        for (int n4 = 0; n4 < 4; ++n4) {
                            const int nt = hh * 4 + n4, bit = nt * 8 + 2 * t;
                            const float b0 = sbias[kb * kBlk + bit], b1 = sbias[kb * kBlk + bit + 1];
                            const float p0 = fast_ex2(fmaf(s[nt][0], sc2, b0) - lse0), p1 = fast_ex2(fmaf(s[nt][1], sc2, b1) - lse0);
                            const float p2 = fast_ex2(fmaf(s[nt][2], sc2, b0) - lse1), p3 = fast_ex2(fmaf(s[nt][3], sc2, b1) - lse1);
                            const float e0 = ((keep_a >> bit) & 1ull) ? dp[n4][0] * ds : 0.f;
                            const float e1 = ((keep_a >> (bit + 1)) & 1ull) ? dp[n4][1] * ds : 0.f;
                            const float e2 = ((keep_c >> bit) & 1ull) ? dp[n4][2] * ds : 0.f;
                            const float e3 = ((keep_c >> (bit + 1)) & 1ull) ? dp[n4][3] * ds : 0.f;
                            s[nt][0] = p0 * (e0 - d0); s[nt][1] = p1 * (e1 - d0);
                            s[nt][2] = p2 * (e2 - d1); s[nt][3] = p3 * (e3 - d1);
                        }
                    }
                    uint32_t dsf[4][4];
                    acc_to_afrag(dsf, s);
                    gemm_nn(dq, dsf, sK + kb * kTileBytes, lane, kvalid);
                }
                store_acc(dbase, ld, row0, len, dq, lane, p.scale, p.scale);
            }
            // ---------------- phase B: dK, dV for key rows row0 .. row0+15 ----------------
            {
                const int ka = row0 + g, kc = ka + 8;
                const float bias0 = sbias[ka], bias1 = sbias[kc];
                float dk[8][4], dv[8][4];
                zero_acc(dk);
                zero_acc(dv);
                for (int qb = 0; qb < nkv; ++qb) {
                    const int qvalid = min(kBlk, len - qb * kBlk);
                    uint32_t af[4][4];
                    float st[8][4];
                    zero_acc(st);
                    load_afrag(af, sK + mytile * kTileBytes, myrow, lane);
                    gemm_nt(st, af, sQ + qb * kTileBytes, lane, qvalid);  // S^T = K Q^T (16 keys x 64 queries)
#pragma unroll
                    for (int nt = 0; nt < 8; ++nt) {
                        const int qi = qb * kBlk + nt * 8 + 2 * t;
                        const float l0 = slse[qi], l1 = slse[qi + 1];
                        st[nt][0] = fast_ex2(fmaf(st[nt][0], sc2, bias0) - l0); st[nt][1] = fast_ex2(fmaf(st[nt][1], sc2, bias0) - l1);
                        st[nt][2] = fast_ex2(fmaf(st[nt][2], sc2, bias1) - l0); st[nt][3] = fast_ex2(fmaf(st[nt][3], sc2, bias1) - l1);
                    }
                    unsigned keepbits = 0xffffffffu;
                    if (drop) {
                        keepbits = 0;
                        // 16-bit slice of the row masks: bit g = key ka, bit 8+g = key kc; keys of this warp = 16*warp..
                        const unsigned short* kp16 = reinterpret_cast<const unsigned short*>(
                            p.keep + (static_cast<unsigned long long>(bh) * np64) * nkb) + warp;
#pragma unroll
                        for (int nt = 0; nt < 8; ++nt) {
                            const long long q = qb * kBlk + nt * 8 + 2 * t;
                            const unsigned w0 = kp16[q * (nkb * 4)], w1 = kp16[(q + 1) * (nkb * 4)];
                            keepbits |= ((w0 >> g) & 1u) << (nt * 4);
                            keepbits |= ((w1 >> g) & 1u) << (nt * 4 + 1);
                            keepbits |= ((w0 >> (8 + g)) & 1u) << (nt * 4 + 2);
                            keepbits |= ((w1 >> (8 + g)) & 1u) << (nt * 4 + 3);
                        }
                    }
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        float w[8];
#pragma unroll
                        for (int e = 0; e < 8; ++e) {
                            const int nt = 2 * jj + (e >> 2), c = e & 3;
                            w[e] = ((keepbits >> (nt * 4 + c)) & 1u) ? st[nt][c] * ds : 0.f;
                        }
                        af[jj][0] = pack_bf16x2(w[0], w[1]); af[jj][1] = pack_bf16x2(w[2], w[3]);
                        af[jj][2] = pack_bf16x2(w[4], w[5]); af[jj][3] = pack_bf16x2(w[6], w[7]);
                    }
                    gemm_nn(dv, af, sdO + qb * kTileBytes, lane, qvalid);  // dV += P_drop^T dO
                    load_afrag(af, sV + mytile * kTileBytes, myrow, lane);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {  // dP^T = V dO^T in two 32-query halves
                        float dpt[4][4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f;
                        gemm_nt_half(dpt, af, sdO + qb * kTileBytes, lane, hh, qvalid);
#pragma unroll
                        for (int n4 = 0; n4 < 4; ++n4) {
                            const int nt = hh * 4 + n4;
                            const int qi = qb * kBlk + nt * 8 + 2 * t;
                            const float dd0 = sD[qi], dd1 = sD[qi + 1];
#pragma unroll
                            for (int c = 0; c < 4; ++c) {
                                const float e = ((keepbits >> (nt * 4 + c)) & 1u) ? dpt[n4][c] * ds : 0.f;
                                st[nt][c] *= e - ((c & 1) ? dd1 : dd0);
                            }
                        }
                    }
                    acc_to_afrag(af, st);
                    gemm_nn(dk, af, sQ + qb * kTileBytes, lane, qvalid);  // dK += dS^T Q
                }
                store_acc(dbase + p.H, ld, row0, len, dk, lane, p.scale, p.scale);
                store_acc(dbase + 2 * p.H, ld, row0, len, dv, lane, 1.f, 1.f);
            }
        }
        __syncthreads();
        if (nbuf == 2) buf ^= 1;
    }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
// These kernels serve 192 < S <= 256 (attn_route): ceil(S / 16) is 13 .. 16 warps, so every launch has 16; warps whose rows
// start past S only help with the loads.
constexpr int kHeadWarps = 16;

template <bool VL>
static int launch_fwd(const AttnParams& p, int nkb, cudaStream_t st) {
    const int smem = 2 * 3 * nkb * kTileBytes + 2 * nkb * kBlk * 4;
    static int configured[kMaxDevices] = {0};
    VB_CHECK_CUDA(ensure_dyn_smem(attn_fwd_head_kernel<kHeadWarps, VL>, smem, configured));
    const int total = p.B * p.A;
    const int grid = total < num_sms() ? total : num_sms();
    ProfScope ps(st, PROF_ATTN_FWD, 4.0 * p.B * p.A * p.S * p.S * kHd, 1);
    VB_CHECK_CUDA(launch_pdl(attn_fwd_head_kernel<kHeadWarps, VL>, dim3(grid), dim3(kHeadWarps * 32), smem, st, p, nkb));
    return 0;
}

// draws the attention-dropout keep bits of the whole layer call (no-op without dropout)
int attn_keep_mask(const AttnParams& p, const AttnDropOffset& off, int nkb, cudaStream_t st) {
    if (p.drop_scale == 0.f) return 0;
    const int np64 = nkb * kBlk;
    const long long nwords = static_cast<long long>(p.B) * p.A * np64 * nkb;
    VB_REQUIRE(nwords * 16 < (1LL << 32), "attention dropout: mask counter space exceeded (B*A*S too large)");
    ProfScope ps(st, PROF_ATTN_FWD, 0.0, 1);
    if (off.offset != nullptr)
        VB_CHECK_CUDA(launch_pdl(attn_keep_mask_off_kernel, dim3(static_cast<unsigned>(nwords / 64)), dim3(64), 0, st, p.keep,
                                 p.keep + nwords, nkb, np64, p.S, off.seed, off.stream_id, off.offset, p.drop_thresh16));
    else
        VB_CHECK_CUDA(launch_pdl(attn_keep_mask_kernel, dim3(static_cast<unsigned>(nwords / 64)), dim3(64), 0, st, p.keep, p.keep + nwords,
                                 nkb, np64, p.S, p.drop_seed, p.drop_thresh16));
    return 0;
}

int attn_fwd_head(const AttnParams& p, const AttnDropOffset& off, int nkb, cudaStream_t st) {
    int rc = attn_keep_mask(p, off, nkb, st);
    if (rc) return rc;
    rc = p.cu_seqlens ? launch_fwd<true>(p, nkb, st) : launch_fwd<false>(p, nkb, st);
    if (rc) return rc;
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <bool VL>
static int launch_bwd(const AttnParams& p, int nkb, cudaStream_t st) {
    const int per_buf = 4 * nkb * kTileBytes + 3 * nkb * kBlk * 4;
    const int nbuf = 2 * per_buf <= 200 * 1024 ? 2 : 1;
    const int smem = nbuf * per_buf;
    static int configured[kMaxDevices] = {0};
    VB_CHECK_CUDA(ensure_dyn_smem(attn_bwd_head_kernel<kHeadWarps, VL>, smem, configured));
    const int total = p.B * p.A;
    const int grid = total < num_sms() ? total : num_sms();
    ProfScope ps(st, PROF_ATTN_DKV, 7.0 * p.B * p.A * p.S * p.S * kHd, 1);
    VB_CHECK_CUDA(launch_pdl(attn_bwd_head_kernel<kHeadWarps, VL>, dim3(grid), dim3(kHeadWarps * 32), smem, st, p, nkb, nbuf));
    return 0;
}

// D[b, h, q] = sum_d dO * O  (the softmax-backward row term), HBM-bound pre-pass shared by the backward kernels
// (varlen: over the `total` packed rows, drow [A, total])
int attn_delta(const AttnParams& p, cudaStream_t st) {
    ProfScope ps(st, PROF_ATTN_DQ, 1.0 * p.B * p.A * p.S * p.S * kHd, 1);
    if (p.cu_seqlens != nullptr) {
        VB_CHECK_CUDA(launch_pdl(attn_delta_kernel<true>, dim3(static_cast<int>((p.total + 7LL) / 8)), dim3(256), 0, st, p.ctx, p.dctx,
                                 p.drow, 1, p.total, p.A, p.H));
        return 0;
    }
    const long long rows = static_cast<long long>(p.B) * p.S;
    VB_CHECK_CUDA(launch_pdl(attn_delta_kernel<false>, dim3(static_cast<int>((rows + 7) / 8)), dim3(256), 0, st, p.ctx, p.dctx, p.drow, p.B,
                             p.S, p.A, p.H));
    return 0;
}

int attn_bwd_head(const AttnParams& p, int nkb, cudaStream_t st, bool delta_ready) {
    if (!delta_ready) {
        int rc0 = attn_delta(p, st);
        if (rc0) return rc0;
    }
    const int rc = p.cu_seqlens ? launch_bwd<true>(p, nkb, st) : launch_bwd<false>(p, nkb, st);
    if (rc) return rc;
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace vb
