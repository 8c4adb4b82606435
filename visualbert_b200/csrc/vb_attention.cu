// vb_attention.cu — fused multi-head self-attention over the [text ; visual] sequence, fwd + bwd.
//
// Replaces BertSelfAttention.forward (reference modeling.py:231-261): scores = QK^T / sqrt(d), then
// + additive mask ((1-mask) * -10000, modeling.py:1293-1294), softmax over keys, dropout on the
// probabilities (modeling.py:251), context = P V, heads merged back to [B*S, H] — without ever
// materialising the [B, A, S, S] score tensor the reference reads/writes five times per layer.
//
// Layout: Q, K, V are column slices of the fused projection output qkv[B*S, 3H] (Q | K | V, head h at
// columns h*64 .. h*64+63 of each third); head_dim is fixed at 64 (BERT-base and -large).
// One CTA = (batch b, head h, 64 query rows); 4 warps x 16 rows; K/V streamed in 64-key blocks through
// a double-buffered, XOR-swizzled shared-memory ring (cp.async); scores, probabilities and the running
// max / sum live in registers (flash-style online softmax in the exp2 domain).
// Backward recomputes P from the saved log-sum-exp: kernel A (per query block) produces dQ and the
// row term D = rowsum(dO * O); kernel B (per key block) produces dK and dV. No atomics, deterministic.
//
// Tensor-core path here is warp-level mma.sync (m16n8k16, bf16 -> fp32); the wgmma kernel of the
// layer is in vb_gemm.cu, where > 96 % of the FLOPs are.
#include "vb_attention.cuh"
#include "vb_internal.h"

namespace vb {

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
// Shared memory: Q tile | K tiles [kMaxSub] | V tiles [kMaxSub]. A "stage" holds up to kMaxSub * 64
// keys; for S <= 256 (every reference config) the whole K/V of the head is resident, all cp.async are
// issued up-front (one commit group per 64-key sub-block) and the warps only wait for the group they
// are about to consume.

// MT = m16 tiles per warp: 1 -> 4 warps x 16 rows, 2 -> 2 warps x 32 rows (FA2-style: each ldmatrix'd K/V
// fragment feeds twice as many MMAs and the warp carries twice as many independent accumulators).
// OFF: the keep bits use the seed folded from p.drop_seed64 + *p.drop_offset (vb_set_dropout_offset)
template <int MT, bool VL, bool OFF>
__device__ __forceinline__ void attn_fwd_body(const AttnParams& p, const int nsub, const unsigned long long* drop_offset = nullptr,
                                              unsigned long long seed64 = 0, unsigned stream_id = 0) {
    constexpr int NT = 128 / MT;
    extern __shared__ __align__(128) uint8_t dsmem[];
    __shared__ float sbias[kMaxSub * kBlk];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const SeqSpan sp = seq_span<VL>(p, b, h);
    const int S = sp.len;  // rows of this sequence
    if (VL && qb * kBlk >= S) return;  // query blocks past the end of a shorter sequence
    const long long ld = 3LL * p.H;
    const bf16* qbase = p.qkv + sp.row0 * ld + h * kHd;
    const bf16* kbase = qbase + p.H;
    const bf16* vbase = qbase + 2 * p.H;
    const uint32_t sQ = smem_u32(dsmem), sK0 = sQ + kTileBytes, sV0 = sK0 + nsub * kTileBytes;
    const int nkb = (p.S + kBlk - 1) / kBlk;      // keep-mask layout: key blocks of the longest sequence
    const int nkv = VL ? (S + kBlk - 1) / kBlk : nkb;  // key blocks of this one

    const float sc2 = p.scale * kLog2e;
    float m[MT][2], l[MT][2];
    float o[MT][8][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
        m[mt][0] = m[mt][1] = -INFINITY;
        l[mt][0] = l[mt][1] = 0.f;
        zero_acc(o[mt]);
    }
    uint32_t qf[MT][4][4];
    const unsigned bh = static_cast<unsigned>(b * p.A + h);
    const int qrow0 = qb * kBlk + warp * 16 * MT;
    const bool active = qrow0 < S;  // warps whose query rows are all padding only help with the loads

    for (int kb0 = 0; kb0 < nkv; kb0 += nsub) {
        const int nb = min(nsub, nkv - kb0);
        if (kb0 > 0) __syncthreads();  // previous stage fully consumed
        if (kb0 == 0) load_tile<NT>(sQ, qbase, ld, qb * kBlk, S, tid);
        for (int j = 0; j < nb; ++j) {
            load_tile<NT>(sK0 + j * kTileBytes, kbase, ld, (kb0 + j) * kBlk, S, tid);
            load_tile<NT>(sV0 + j * kTileBytes, vbase, ld, (kb0 + j) * kBlk, S, tid);
            cp_async_commit();
        }
        for (int i = tid; i < nb * kBlk; i += NT) {
            const int key = kb0 * kBlk + i;
            sbias[i] = key_bias2<VL>(p, b, key, S);
        }
        for (int j = 0; j < nb; ++j) {
            cp_async_wait_dyn(nb - 1 - j);
            __syncthreads();
            if (!active) continue;
            if (kb0 == 0 && j == 0) {
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) load_afrag(qf[mt], sQ, warp * 16 * MT + mt * 16, lane);
            }
            const int kb = kb0 + j;
            const int kvalid = min(kBlk, S - kb * kBlk);
            float s[MT][8][4];
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) zero_acc(s[mt]);
            gemm_nt_mt<MT>(s, qf, sK0 + j * kTileBytes, lane, kvalid);
            uint32_t pf[MT][4][4];
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const float b0 = sbias[j * kBlk + nt * 8 + 2 * t], b1 = sbias[j * kBlk + nt * 8 + 2 * t + 1];
                    s[mt][nt][0] = fmaf(s[mt][nt][0], sc2, b0); s[mt][nt][1] = fmaf(s[mt][nt][1], sc2, b1);
                    s[mt][nt][2] = fmaf(s[mt][nt][2], sc2, b0); s[mt][nt][3] = fmaf(s[mt][nt][3], sc2, b1);
                    mx[0] = fmaxf(mx[0], fmaxf(s[mt][nt][0], s[mt][nt][1]));
                    mx[1] = fmaxf(mx[1], fmaxf(s[mt][nt][2], s[mt][nt][3]));
                }
                float alpha[2];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
                    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
                    const float mn = fmaxf(m[mt][r], mx[r]);
                    alpha[r] = fast_ex2(m[mt][r] - mn);
                    m[mt][r] = mn;
                }
                float rs[2] = {0.f, 0.f};
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    s[mt][nt][0] = fast_ex2(s[mt][nt][0] - m[mt][0]); s[mt][nt][1] = fast_ex2(s[mt][nt][1] - m[mt][0]);
                    s[mt][nt][2] = fast_ex2(s[mt][nt][2] - m[mt][1]); s[mt][nt][3] = fast_ex2(s[mt][nt][3] - m[mt][1]);
                    rs[0] += s[mt][nt][0] + s[mt][nt][1];
                    rs[1] += s[mt][nt][2] + s[mt][nt][3];
                }
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
                    rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
                    l[mt][r] = l[mt][r] * alpha[r] + rs[r];
                }
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    o[mt][nt][0] *= alpha[0]; o[mt][nt][1] *= alpha[0];
                    o[mt][nt][2] *= alpha[1]; o[mt][nt][3] *= alpha[1];
                }
                if (p.drop_scale != 0.f) {
                    const int qa = qrow0 + mt * 16 + g, qc = qa + 8;
                    const unsigned sd = OFF ? attn_seed_fold(seed64 + *drop_offset, stream_id) : p.drop_seed;
                    const uint32_t ka_bits = attn_keep16(sd, bh, qa, kb, t, nkb, p.drop_thresh16);
                    const uint32_t kc_bits = attn_keep16(sd, bh, qc, kb, t, nkb, p.drop_thresh16);
#pragma unroll
                    for (int nt = 0; nt < 8; ++nt) {
                        s[mt][nt][0] = ((ka_bits >> (2 * nt)) & 1u) ? s[mt][nt][0] * p.drop_scale : 0.f;
                        s[mt][nt][1] = ((ka_bits >> (2 * nt + 1)) & 1u) ? s[mt][nt][1] * p.drop_scale : 0.f;
                        s[mt][nt][2] = ((kc_bits >> (2 * nt)) & 1u) ? s[mt][nt][2] * p.drop_scale : 0.f;
                        s[mt][nt][3] = ((kc_bits >> (2 * nt + 1)) & 1u) ? s[mt][nt][3] * p.drop_scale : 0.f;
                    }
                    const unsigned long long ma = quad_mask64(ka_bits, t), mc = quad_mask64(kc_bits, t);
                    if (t == 0) {  // rows are padded to nkb*64 in the mask buffer: no bounds check needed
                        unsigned long long* kp = p.keep + (static_cast<unsigned long long>(bh) * (nkb * kBlk)) * nkb;
                        kp[static_cast<long long>(qa) * nkb + kb] = ma;
                        kp[static_cast<long long>(qc) * nkb + kb] = mc;
                    }
                }
                acc_to_afrag(pf[mt], s[mt]);
            }
            gemm_nn_mt<MT>(o, pf, sV0 + j * kTileBytes, lane, kvalid);
        }
    }
    if (!active) return;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
        const int r0 = qrow0 + mt * 16;
        const float inv0 = 1.f / l[mt][0], inv1 = 1.f / l[mt][1];
        store_acc(p.ctx + sp.row0 * p.H + h * kHd, p.H, r0, S, o[mt], lane, inv0, inv1);
        if (t == 0 && p.lse != nullptr) {
            float* lse = p.lse + sp.stat0;
            if (r0 + g < S) lse[r0 + g] = (m[mt][0] + log2f(l[mt][0])) * 0.6931471805599453f;
            if (r0 + g + 8 < S) lse[r0 + g + 8] = (m[mt][1] + log2f(l[mt][1])) * 0.6931471805599453f;
        }
    }
}

template <int MT, int MINB, bool VL = false>
__global__ void __launch_bounds__(128 / MT, MINB) attn_fwd_kernel(const AttnParams p, const int nsub) { attn_fwd_body<MT, VL, false>(p, nsub); }
template <int MT, int MINB, bool VL = false>
__global__ void __launch_bounds__(128 / MT, MINB)
attn_fwd_off_kernel(const AttnParams p, const int nsub, const unsigned long long* drop_offset, unsigned long long seed64, unsigned stream_id) {
    attn_fwd_body<MT, VL, true>(p, nsub, drop_offset, seed64, stream_id);
}

// ------------------------------------------------------------------------------------------------
// backward A: per query block — D = rowsum(dO * O), dQ = scale * sum_k dS K
// Shared memory: Q | dO | O | K tiles [nsub] | V tiles [nsub]
// ------------------------------------------------------------------------------------------------
template <int MINB, bool VL = false>
__global__ void __launch_bounds__(128, MINB)
attn_bwd_dq_kernel(const AttnParams p, const int nsub) {
    extern __shared__ __align__(128) uint8_t dsmem[];
    __shared__ float sbias[kMaxSub * kBlk];
    __shared__ float sD[kBlk];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const SeqSpan sp = seq_span<VL>(p, b, h);
    const int S = sp.len;
    if (VL && qb * kBlk >= S) return;
    const long long ld = 3LL * p.H;
    const bf16* qbase = p.qkv + sp.row0 * ld + h * kHd;
    const bf16* kbase = qbase + p.H;
    const bf16* vbase = qbase + 2 * p.H;
    const bf16* obase = p.ctx + sp.row0 * p.H + h * kHd;
    const bf16* dobase = p.dctx + sp.row0 * p.H + h * kHd;
    const uint32_t sQ = smem_u32(dsmem), sdO = sQ + kTileBytes, sO = sQ + 2 * kTileBytes;
    const uint32_t sK0 = sQ + 3 * kTileBytes, sV0 = sK0 + nsub * kTileBytes;
    const int nkb = (p.S + kBlk - 1) / kBlk;
    const int nkv = VL ? (S + kBlk - 1) / kBlk : nkb;
    const int qrow0 = qb * kBlk + warp * 16;
    const bool active = qrow0 < S;
    const float* lsep = p.lse + sp.stat0;
    const float lse0 = (qrow0 + g < S) ? lsep[qrow0 + g] * kLog2e : 0.f;
    const float lse1 = (qrow0 + g + 8 < S) ? lsep[qrow0 + g + 8] * kLog2e : 0.f;
    const float sc2 = p.scale * kLog2e;
    const unsigned bh = static_cast<unsigned>(b * p.A + h);
    uint32_t qf[4][4], dof[4][4];
    float d0 = 0.f, d1 = 0.f;
    float dq[8][4];
    zero_acc(dq);

    for (int kb0 = 0; kb0 < nkv; kb0 += nsub) {
        const int nb = min(nsub, nkv - kb0);
        if (kb0 > 0) __syncthreads();
        if (kb0 == 0) {
            load_tile(sQ, qbase, ld, qb * kBlk, S, tid);
            load_tile(sdO, dobase, p.H, qb * kBlk, S, tid);
            load_tile(sO, obase, p.H, qb * kBlk, S, tid);
        }
        for (int j = 0; j < nb; ++j) {
            load_tile(sK0 + j * kTileBytes, kbase, ld, (kb0 + j) * kBlk, S, tid);
            load_tile(sV0 + j * kTileBytes, vbase, ld, (kb0 + j) * kBlk, S, tid);
            cp_async_commit();
        }
        for (int i = tid; i < nb * kBlk; i += 128) {
            const int key = kb0 * kBlk + i;
            sbias[i] = key_bias2<VL>(p, b, key, S);
        }
        for (int j = 0; j < nb; ++j) {
            cp_async_wait_dyn(nb - 1 - j);
            __syncthreads();
            if (kb0 == 0 && j == 0) {
                // D[row] = sum_d dO * O : two threads per row (block-wide, then one more barrier)
                const int r = tid >> 1, half = tid & 1;
                float acc = 0.f;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int chunk = half * 4 + c;
                    const uint4 a = *reinterpret_cast<const uint4*>(dsmem + kTileBytes + swz(r, chunk));
                    const uint4 ov = *reinterpret_cast<const uint4*>(dsmem + 2 * kTileBytes + swz(r, chunk));
                    const uint32_t av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float2 x = unpack_bf16x2(av[i]), y = unpack_bf16x2(bv[i]);
                        acc += x.x * y.x + x.y * y.y;
                    }
                }
                acc += __shfl_xor_sync(0xffffffffu, acc, 1);
                if (half == 0) {
                    sD[r] = acc;
                    const int q = qb * kBlk + r;
                    if (q < S) p.drow[sp.stat0 + q] = acc;
                }
                __syncthreads();
                if (active) {
                    load_afrag(qf, sQ, warp * 16, lane);
                    load_afrag(dof, sdO, warp * 16, lane);
                    d0 = sD[warp * 16 + g];
                    d1 = sD[warp * 16 + g + 8];
                }
            }
            if (!active) continue;
            const int kb = kb0 + j;
            const int kvalid = min(kBlk, S - kb * kBlk);
            float s[8][4];
            zero_acc(s);
            unsigned long long keep_a = 0, keep_c = 0;
            if (p.drop_scale != 0.f) {
                const unsigned long long* kp = p.keep + (static_cast<unsigned long long>(bh) * (nkb * kBlk)) * nkb;
                keep_a = kp[static_cast<long long>(qrow0 + g) * nkb + kb];
                keep_c = kp[static_cast<long long>(qrow0 + g + 8) * nkb + kb];
            }
            gemm_nt(s, qf, sK0 + j * kTileBytes, lane, kvalid);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {  // dP = dO V^T in two 32-key halves (register pressure)
                float dp[4][4];
#pragma unroll
                for (int i = 0; i < 4; ++i) dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
                gemm_nt_half(dp, dof, sV0 + j * kTileBytes, lane, hh, kvalid);
#pragma unroll
                for (int n4 = 0; n4 < 4; ++n4) {
                    const int nt = hh * 4 + n4;
                    const float b0 = sbias[j * kBlk + nt * 8 + 2 * t], b1 = sbias[j * kBlk + nt * 8 + 2 * t + 1];
                    const float p0 = fast_ex2(fmaf(s[nt][0], sc2, b0) - lse0), p1 = fast_ex2(fmaf(s[nt][1], sc2, b1) - lse0);
                    const float p2 = fast_ex2(fmaf(s[nt][2], sc2, b0) - lse1), p3 = fast_ex2(fmaf(s[nt][3], sc2, b1) - lse1);
                    float e0 = dp[n4][0], e1 = dp[n4][1], e2 = dp[n4][2], e3 = dp[n4][3];
                    if (p.drop_scale != 0.f) {
                        const int bit = nt * 8 + 2 * t;
                        e0 = ((keep_a >> bit) & 1ull) ? e0 * p.drop_scale : 0.f;
                        e1 = ((keep_a >> (bit + 1)) & 1ull) ? e1 * p.drop_scale : 0.f;
                        e2 = ((keep_c >> bit) & 1ull) ? e2 * p.drop_scale : 0.f;
                        e3 = ((keep_c >> (bit + 1)) & 1ull) ? e3 * p.drop_scale : 0.f;
                    }
                    s[nt][0] = p0 * (e0 - d0); s[nt][1] = p1 * (e1 - d0);
                    s[nt][2] = p2 * (e2 - d1); s[nt][3] = p3 * (e3 - d1);
                }
            }
            uint32_t dsf[4][4];
            acc_to_afrag(dsf, s);
            gemm_nn(dq, dsf, sK0 + j * kTileBytes, lane, kvalid);
        }
    }
    if (!active) return;
    store_acc(p.dqkv + sp.row0 * ld + h * kHd, ld, qrow0, S, dq, lane, p.scale, p.scale);
}

// ------------------------------------------------------------------------------------------------
// backward B: per key block — dV = P_drop^T dO, dK = scale * dS^T Q
// Shared memory: K | V | Q tiles [nsub] | dO tiles [nsub]; K/V fragments are re-read from shared memory
// per query block instead of being pinned in 32 registers.
// ------------------------------------------------------------------------------------------------
template <int MINB, bool VL = false>
__global__ void __launch_bounds__(128, MINB)
attn_bwd_dkv_kernel(const AttnParams p, const int nsub) {
    extern __shared__ __align__(128) uint8_t dsmem[];
    __shared__ float slse[kMaxSub * kBlk];
    __shared__ float sD[kMaxSub * kBlk];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int kbk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const SeqSpan sp = seq_span<VL>(p, b, h);
    const int S = sp.len;
    if (VL && kbk * kBlk >= S) return;  // key blocks past the end of a shorter sequence
    const long long ld = 3LL * p.H;
    const bf16* qbase = p.qkv + sp.row0 * ld + h * kHd;
    const bf16* kbase = qbase + p.H;
    const bf16* vbase = qbase + 2 * p.H;
    const bf16* dobase = p.dctx + sp.row0 * p.H + h * kHd;
    const uint32_t sK = smem_u32(dsmem), sV = sK + kTileBytes, sQ0 = sK + 2 * kTileBytes, sdO0 = sQ0 + nsub * kTileBytes;
    const int nqb = (p.S + kBlk - 1) / kBlk;            // keep-mask layout
    const int nqv = VL ? (S + kBlk - 1) / kBlk : nqb;  // query blocks of this sequence
    const float* lsep = p.lse + sp.stat0;
    const float* drp = p.drow + sp.stat0;
    const int krow0 = kbk * kBlk + warp * 16;
    const bool active = krow0 < S;
    const int ka = krow0 + g, kc = krow0 + g + 8;
    const float bias0 = key_bias2<VL>(p, b, ka, S);
    const float bias1 = key_bias2<VL>(p, b, kc, S);
    const float sc2 = p.scale * kLog2e;
    const unsigned bh = static_cast<unsigned>(b * p.A + h);
    float dk[8][4], dv[8][4];
    zero_acc(dk);
    zero_acc(dv);

    for (int qb0 = 0; qb0 < nqv; qb0 += nsub) {
        const int nb = min(nsub, nqv - qb0);
        if (qb0 > 0) __syncthreads();
        if (qb0 == 0) {
            load_tile(sK, kbase, ld, kbk * kBlk, S, tid);
            load_tile(sV, vbase, ld, kbk * kBlk, S, tid);
        }
        for (int j = 0; j < nb; ++j) {
            load_tile(sQ0 + j * kTileBytes, qbase, ld, (qb0 + j) * kBlk, S, tid);
            load_tile(sdO0 + j * kTileBytes, dobase, p.H, (qb0 + j) * kBlk, S, tid);
            cp_async_commit();
        }
        for (int i = tid; i < nb * kBlk; i += 128) {
            const int q = qb0 * kBlk + i;
            slse[i] = q < S ? lsep[q] * kLog2e : INFINITY;  // +inf => p = 0 for padded queries
            sD[i] = q < S ? drp[q] : 0.f;
        }
        for (int j = 0; j < nb; ++j) {
            cp_async_wait_dyn(nb - 1 - j);
            __syncthreads();
            if (!active) continue;
            const int qb = qb0 + j;
            const int qvalid = min(kBlk, S - qb * kBlk);
            uint32_t af[4][4];
            float st[8][4];
            zero_acc(st);
            load_afrag(af, sK, warp * 16, lane);
            gemm_nt(st, af, sQ0 + j * kTileBytes, lane, qvalid);  // S^T = K Q^T (16 keys x 64 queries)
            // probabilities (st := P^T); dropped copy -> A fragments of the dV GEMM
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const int qi = nt * 8 + 2 * t;
                const float l0 = slse[j * kBlk + qi], l1 = slse[j * kBlk + qi + 1];
                st[nt][0] = fast_ex2(fmaf(st[nt][0], sc2, bias0) - l0); st[nt][1] = fast_ex2(fmaf(st[nt][1], sc2, bias0) - l1);
                st[nt][2] = fast_ex2(fmaf(st[nt][2], sc2, bias1) - l0); st[nt][3] = fast_ex2(fmaf(st[nt][3], sc2, bias1) - l1);
            }
            unsigned keepbits = 0xffffffffu;
            if (p.drop_scale != 0.f) {
                keepbits = 0;
#pragma unroll
                // 16-bit slice of the row masks: bit g = key ka, bit 8+g = key kc (= ka + 8)
                const unsigned short* kp16 = reinterpret_cast<const unsigned short*>(
                    p.keep + (static_cast<unsigned long long>(bh) * (nqb * kBlk)) * nqb) + kbk * 4 + warp;
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const long long q = qb * kBlk + nt * 8 + 2 * t;
                    const unsigned w0 = kp16[q * (nqb * 4)], w1 = kp16[(q + 1) * (nqb * 4)];
                    keepbits |= ((w0 >> g) & 1u) << (nt * 4);
                    keepbits |= ((w1 >> g) & 1u) << (nt * 4 + 1);
                    keepbits |= ((w0 >> (8 + g)) & 1u) << (nt * 4 + 2);
                    keepbits |= ((w1 >> (8 + g)) & 1u) << (nt * 4 + 3);
                }
            }
            const float ds = p.drop_scale != 0.f ? p.drop_scale : 1.f;
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
            gemm_nn(dv, af, sdO0 + j * kTileBytes, lane, qvalid);  // dV += P_drop^T dO
            load_afrag(af, sV, warp * 16, lane);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {  // dP^T = V dO^T in two 32-query halves (register pressure)
                float dpt[4][4];
#pragma unroll
                for (int i = 0; i < 4; ++i) dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f;
                gemm_nt_half(dpt, af, sdO0 + j * kTileBytes, lane, hh, qvalid);
#pragma unroll
                for (int n4 = 0; n4 < 4; ++n4) {
                    const int nt = hh * 4 + n4;
                    const int qi = nt * 8 + 2 * t;
                    const float dd0 = sD[j * kBlk + qi], dd1 = sD[j * kBlk + qi + 1];
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const float e = ((keepbits >> (nt * 4 + c)) & 1u) ? dpt[n4][c] * ds : 0.f;
                        st[nt][c] *= e - ((c & 1) ? dd1 : dd0);
                    }
                }
            }
            acc_to_afrag(af, st);
            gemm_nn(dk, af, sQ0 + j * kTileBytes, lane, qvalid);  // dK += dS^T Q
        }
    }
    if (!active) return;
    bf16* dbase = p.dqkv + sp.row0 * ld + h * kHd;
    store_acc(dbase + p.H, ld, krow0, S, dk, lane, p.scale, p.scale);
    store_acc(dbase + 2 * p.H, ld, krow0, S, dv, lane, 1.f, 1.f);
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
static bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

static int fill_params(AttnParams& p, const void* qkv, const float* mask_bias, void* ctx, float* lse,
                       const void* dctx, void* dqkv, float* drow, void* keep, int B, int S, int A, int H,
                       float dropout_p, unsigned long long seed, unsigned stream_id, AttnDropOffset* off = nullptr) {
    VB_REQUIRE(B > 0 && S > 0 && A > 0, "attention: empty problem");
    VB_REQUIRE(H == A * kHd, "attention: head_dim must be 64 (hidden=%d heads=%d)", H, A);
    VB_REQUIRE(A <= 65535 && B <= 65535, "attention: grid too large");
    VB_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "attention: dropout_p out of range");
    VB_REQUIRE(dropout_p == 0.f || keep != nullptr, "attention: dropout needs the keep-mask buffer (vb_attention_keep_bytes)");
    // every route reads qkv, and in the backward ctx and dctx, in 16-byte pieces (TMA, cp.async, vector loads)
    VB_REQUIRE(aligned16(qkv) && (dctx == nullptr || (aligned16(ctx) && aligned16(dctx))),
               "attention: qkv, ctx (backward) and dctx must be 16-byte aligned");
    p.keep = static_cast<unsigned long long*>(keep);
    p.qkv = static_cast<const bf16*>(qkv);
    p.mask_bias = mask_bias;
    p.ctx = static_cast<bf16*>(ctx);
    p.lse = lse;
    p.dctx = static_cast<const bf16*>(dctx);
    p.dqkv = static_cast<bf16*>(dqkv);
    p.drow = drow;
    p.B = B; p.S = S; p.A = A; p.H = H;
    p.cu_seqlens = nullptr;
    p.total = 0;
    p.scale = 0.125f;
    // 8-bit quantised keep threshold (see attn_hash); the scale uses the quantised probability
    const unsigned th8 = static_cast<unsigned>(dropout_p * 256.f + 0.5f);
    p.drop_thresh16 = th8;
    p.drop_scale = dropout_p > 0.f ? 256.f / (256.f - static_cast<float>(th8 > 255 ? 255 : th8)) : 0.f;
    // fold the per-layer stream id into the 32-bit seed of the element hash (on the device when the offset is there)
    p.drop_seed = attn_seed_fold(seed, stream_id);
    if (off != nullptr) *off = AttnDropOffset{dropout_p > 0.f ? drop_offset() : nullptr, seed, stream_id};
    return 0;
}

long long attn_keep_bytes(int B, int S, int A) {
    const long long nkb = (S + kBlk - 1) / kBlk;
    return 2 * static_cast<long long>(B) * A * (nkb * kBlk) * nkb * 8;  // query-major words + their transpose (key-major)
}

// variable-length calls: the sequence table and the packed row count (what can be checked without reading device memory)
static int set_varlen(AttnParams& p, const int* cu_seqlens, int total, const void* qkv, const void* out) {
    VB_REQUIRE(cu_seqlens != nullptr, "attention varlen: cu_seqlens is NULL");
    VB_REQUIRE(total >= 0, "attention varlen: total (%d) must be >= 0", total);
    VB_REQUIRE(qkv != nullptr && out != nullptr, "attention varlen: null pointer");
    VB_REQUIRE(static_cast<long long>(p.A) * total < (1LL << 31), "attention varlen: heads * total too large");
    p.cu_seqlens = cu_seqlens;
    p.total = total;
    return 0;
}

static int attn_fwd_launch(const AttnParams& p, const AttnDropOffset& off, cudaStream_t st) {
    const int B = p.B, S = p.S, A = p.A;
    dim3 grid((S + kBlk - 1) / kBlk, A, B);
    const AttnRoute route = attn_route(S);
    if (route == AttnRoute::Wgmma) return attn_fwd_wgmma(p, off, st);
    if (route == AttnRoute::Head) return attn_fwd_head(p, off, static_cast<int>(grid.x), st);
    const long long nkb = grid.x;
    VB_REQUIRE(p.drop_scale == 0.f || static_cast<long long>(B) * A * (nkb * kBlk) * nkb * 16 < (1LL << 32),
               "attention dropout: mask counter space exceeded (B*A*S too large)");
    const int nsub = static_cast<int>(grid.x) < kMaxSub ? static_cast<int>(grid.x) : kMaxSub;
    const int smem = (1 + 2 * nsub) * kTileBytes;
    static int configured[kMaxDevices] = {0}, configured_vl[kMaxDevices] = {0};
    static int configured_off[kMaxDevices] = {0}, configured_vl_off[kMaxDevices] = {0};
    {
        ProfScope ps(st, PROF_ATTN_FWD, 4.0 * B * A * S * S * kHd, 1);
        if (off.offset != nullptr && p.cu_seqlens == nullptr) {
            VB_CHECK_CUDA(ensure_dyn_smem(attn_fwd_off_kernel<1, 3>, (1 + 2 * kMaxSub) * kTileBytes, configured_off));
            attn_fwd_off_kernel<1, 3><<<grid, 128, smem, st>>>(p, nsub, off.offset, off.seed, off.stream_id);
        } else if (off.offset != nullptr) {
            VB_CHECK_CUDA(ensure_dyn_smem(attn_fwd_off_kernel<1, 3, true>, (1 + 2 * kMaxSub) * kTileBytes, configured_vl_off));
            attn_fwd_off_kernel<1, 3, true><<<grid, 128, smem, st>>>(p, nsub, off.offset, off.seed, off.stream_id);
        } else if (p.cu_seqlens == nullptr) {
            VB_CHECK_CUDA(ensure_dyn_smem(attn_fwd_kernel<1, 3>, (1 + 2 * kMaxSub) * kTileBytes, configured));
            attn_fwd_kernel<1, 3><<<grid, 128, smem, st>>>(p, nsub);
        } else {
            VB_CHECK_CUDA(ensure_dyn_smem(attn_fwd_kernel<1, 3, true>, (1 + 2 * kMaxSub) * kTileBytes, configured_vl));
            attn_fwd_kernel<1, 3, true><<<grid, 128, smem, st>>>(p, nsub);
        }
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int attn_fwd(const void* qkv, const float* mask_bias, void* ctx, float* lse, void* keep, int B, int S, int A, int H,
             float dropout_p, unsigned long long seed, unsigned stream_id, cudaStream_t st) {
    AttnParams p;
    AttnDropOffset off;
    int rc = fill_params(p, qkv, mask_bias, ctx, lse, nullptr, nullptr, nullptr, keep, B, S, A, H, dropout_p, seed, stream_id, &off);
    if (rc) return rc;
    return attn_fwd_launch(p, off, st);
}

int attn_fwd_varlen(const void* qkv, const int* cu_seqlens, void* ctx, float* lse, void* keep, int B, int max_seq, int total,
                    int A, int H, float dropout_p, unsigned long long seed, unsigned stream_id, cudaStream_t st, bool need_lse) {
    AttnParams p;
    AttnDropOffset off;
    int rc = fill_params(p, qkv, nullptr, ctx, lse, nullptr, nullptr, nullptr, keep, B, max_seq, A, H, dropout_p, seed, stream_id, &off);
    if (rc) return rc;
    VB_REQUIRE(lse != nullptr || !need_lse, "attention varlen: lse is NULL");
    if ((rc = set_varlen(p, cu_seqlens, total, qkv, ctx))) return rc;
    if (total == 0) return 0;  // no rows: nothing to compute or store
    return attn_fwd_launch(p, off, st);
}

static int attn_bwd_launch(const AttnParams& p, cudaStream_t st, bool delta_ready) {
    const int B = p.B, S = p.S, A = p.A;
    dim3 grid((S + kBlk - 1) / kBlk, A, B);
    const AttnRoute route = attn_route(S);
    if (route == AttnRoute::Wgmma) return attn_bwd_wgmma(p, st, delta_ready);
    if (route == AttnRoute::Head) return attn_bwd_head(p, static_cast<int>(grid.x), st, delta_ready);
    const int nsub = static_cast<int>(grid.x) < kMaxSub ? static_cast<int>(grid.x) : kMaxSub;
    const bool vl = p.cu_seqlens != nullptr;
    static int c0[kMaxDevices] = {0}, c1[kMaxDevices] = {0}, v0[kMaxDevices] = {0}, v1[kMaxDevices] = {0};
    if (vl) {
        VB_CHECK_CUDA(ensure_dyn_smem(attn_bwd_dq_kernel<3, true>, (3 + 2 * kMaxSub) * kTileBytes, v0));
        VB_CHECK_CUDA(ensure_dyn_smem(attn_bwd_dkv_kernel<3, true>, (2 + 2 * kMaxSub) * kTileBytes, v1));
    } else {
        VB_CHECK_CUDA(ensure_dyn_smem(attn_bwd_dq_kernel<3>, (3 + 2 * kMaxSub) * kTileBytes, c0));
        VB_CHECK_CUDA(ensure_dyn_smem(attn_bwd_dkv_kernel<3>, (2 + 2 * kMaxSub) * kTileBytes, c1));
    }
    {   // algorithmic work of the backward = 2x forward (recompute not credited), split evenly over the two kernels
        ProfScope ps(st, PROF_ATTN_DQ, 4.0 * B * A * S * S * kHd, 1);
        if (vl) attn_bwd_dq_kernel<3, true><<<grid, 128, (3 + 2 * nsub) * kTileBytes, st>>>(p, nsub);
        else attn_bwd_dq_kernel<3><<<grid, 128, (3 + 2 * nsub) * kTileBytes, st>>>(p, nsub);
    }
    {
        ProfScope ps(st, PROF_ATTN_DKV, 4.0 * B * A * S * S * kHd, 1);
        if (vl) attn_bwd_dkv_kernel<3, true><<<grid, 128, (2 + 2 * nsub) * kTileBytes, st>>>(p, nsub);
        else attn_bwd_dkv_kernel<3><<<grid, 128, (2 + 2 * nsub) * kTileBytes, st>>>(p, nsub);
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int attn_bwd(const void* qkv, const float* mask_bias, const void* ctx, const float* lse, const void* keep,
             const void* dctx, void* dqkv, float* drow, int B, int S, int A, int H, float dropout_p,
             unsigned long long seed, unsigned stream_id, cudaStream_t st, bool delta_ready) {
    AttnParams p;
    int rc = fill_params(p, qkv, mask_bias, const_cast<void*>(ctx), const_cast<float*>(lse), dctx, dqkv, drow,
                         const_cast<void*>(keep), B, S, A, H, dropout_p, seed, stream_id);
    if (rc) return rc;
    return attn_bwd_launch(p, st, delta_ready);
}

int attn_bwd_varlen(const void* qkv, const int* cu_seqlens, const void* ctx, const float* lse, const void* keep,
                    const void* dctx, void* dqkv, float* drow, int B, int max_seq, int total, int A, int H, float dropout_p,
                    unsigned long long seed, unsigned stream_id, cudaStream_t st, bool delta_ready) {
    AttnParams p;
    int rc = fill_params(p, qkv, nullptr, const_cast<void*>(ctx), const_cast<float*>(lse), dctx, dqkv, drow,
                         const_cast<void*>(keep), B, max_seq, A, H, dropout_p, seed, stream_id);
    if (rc) return rc;
    VB_REQUIRE(ctx && lse && dctx && drow, "attention varlen: null pointer");
    if ((rc = set_varlen(p, cu_seqlens, total, qkv, dqkv))) return rc;
    if (total == 0) return 0;
    return attn_bwd_launch(p, st, delta_ready);
}

}  // namespace vb

extern "C" {
int64_t vb_attention_keep_bytes(int32_t batch, int32_t seq, int32_t heads) {
    return vb::attn_keep_bytes(batch, seq, heads);
}
int vb_attention_fwd(const void* qkv, const float* mask_bias, void* ctx, float* lse, void* keep_mask, int32_t batch,
                     int32_t seq, int32_t heads, int32_t hidden, float dropout_p, uint64_t dropout_seed,
                     uint32_t dropout_stream, void* stream) {
    return vb::attn_fwd(qkv, mask_bias, ctx, lse, keep_mask, batch, seq, heads, hidden, dropout_p, dropout_seed,
                        dropout_stream, static_cast<cudaStream_t>(stream));
}
int vb_attention_bwd(const void* qkv, const float* mask_bias, const void* ctx, const float* lse, const void* keep_mask,
                     const void* dctx, void* dqkv, float* drow, int32_t batch, int32_t seq, int32_t heads,
                     int32_t hidden, float dropout_p, uint64_t dropout_seed, uint32_t dropout_stream, void* stream) {
    return vb::attn_bwd(qkv, mask_bias, ctx, lse, keep_mask, dctx, dqkv, drow, batch, seq, heads, hidden, dropout_p,
                        dropout_seed, dropout_stream, static_cast<cudaStream_t>(stream), false);
}
int vb_attention_fwd_varlen(const void* qkv, const int32_t* cu_seqlens, void* ctx, float* lse, void* keep_mask, int32_t batch,
                            int32_t max_seq, int32_t total, int32_t heads, int32_t hidden, float dropout_p, uint64_t dropout_seed,
                            uint32_t dropout_stream, void* stream) {
    return vb::attn_fwd_varlen(qkv, cu_seqlens, ctx, lse, keep_mask, batch, max_seq, total, heads, hidden, dropout_p, dropout_seed,
                               dropout_stream, static_cast<cudaStream_t>(stream));
}
int vb_attention_bwd_varlen(const void* qkv, const int32_t* cu_seqlens, const void* ctx, const float* lse, const void* keep_mask,
                            const void* dctx, void* dqkv, float* drow, int32_t batch, int32_t max_seq, int32_t total, int32_t heads,
                            int32_t hidden, float dropout_p, uint64_t dropout_seed, uint32_t dropout_stream, void* stream) {
    return vb::attn_bwd_varlen(qkv, cu_seqlens, ctx, lse, keep_mask, dctx, dqkv, drow, batch, max_seq, total, heads, hidden,
                               dropout_p, dropout_seed, dropout_stream, static_cast<cudaStream_t>(stream), false);
}
}
