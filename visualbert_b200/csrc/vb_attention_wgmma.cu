// vb_attention_wgmma.cu — Hopper attention forward and backward for seq <= 192 (every reference config).
//
// One CTA per (batch, head), NKB = ceil(S / 64) warpgroups (one per 64-row block of the sequence). One thread loads the
// head's Q, K, V (and dO) 64 x 64 tiles with TMA (128B swizzle, completion on one mbarrier); all contractions are
// wgmma.mma_async 64 x 64 x 16:
//   forward   S = Q K^T (both operands from shared memory), softmax of whole rows in registers (no online rescaling: a
//             warpgroup holds all keys of its 64 queries), dropout from the layer's keep-mask words, O = P V with P handed
//             to the MMA as register fragments (the accumulator layout of S is the A-fragment layout of P).
//   backward  P is recomputed from the saved log-sum-exp. Pass 1: P_drop -> shared memory, then each warpgroup computes dV of
//             its 64 keys as P_drop^T dO (A read transposed from shared memory). Pass 2: dP = dO V^T, dS = P (dP_drop - D),
//             dQ += dS K from registers, dS -> shared memory, then dK = dS^T Q per key block. D = rowsum(dO * O) comes from
//             the epilogue of the GEMM that produced dO, or from attn_delta.
// Rows and keys >= S inside the last 64-row tile: keys get a -inf bias (probability 0), queries are never stored and, in
// the backward, get lse = +inf (probability 0), so whatever the tile holds there contributes nothing.
// Variable-length calls (VL): the CTA of (b, h) loads the packed rows cu[b] + 64 kb .. from a tensor map of `total` rows, only
// for the key blocks kb < ceil(len / 64) of its own sequence. Tile rows past len belong to the next sequence (or are TMA's
// zero fill past `total`): the same -inf bias / +inf lse rule makes them contribute nothing, and no ctx, dQ, dK or dV row past
// len is stored. Warpgroups whose 64-row block starts past len issue no MMAs.
#include "vb_attention.cuh"

namespace vb {

constexpr int kWgTile = kBlk * kHd * 2;   // one 64 x 64 bf16 tile, 128B-swizzled rows (8 KB)

template <int NKB>
struct AttnSmem {
    static constexpr int FWD_BYTES = 3 * NKB * kWgTile + NKB * kBlk * 4 + 16 + 1024;
    static constexpr int BWD_BYTES = (4 * NKB + NKB * NKB) * kWgTile + NKB * kBlk * 4 + 16 + 1024;
};

__device__ __forceinline__ uint64_t tile_desc(uint32_t saddr) { return wgmma_desc_sw128(saddr, kWgTile, 1024); }

// keep bits of query row q for key block kb, shifted so that the bits of this lane's columns (8 j + 2 t + c) sit at 8 j + c
__device__ __forceinline__ unsigned long long keep_word(const AttnParams& p, unsigned bh, int q, int kb, int nkb, int t) {
    if (p.drop_scale == 0.f) return ~0ull;
    return p.keep[(static_cast<unsigned long long>(bh) * (nkb * kBlk) + q) * nkb + kb] >> (2 * t);
}

// S (64 x 64 per key block) = Q_wg K_kb^T, raw dot products
template <int NKB>
__device__ __forceinline__ void qk_block(float (&s)[32], uint32_t sQ, uint32_t sK, int wg, int kb) {
#pragma unroll
    for (int k = 0; k < kHd / 16; ++k)
        wgmma_m64n64k16_ss<0, 0>(s, tile_desc(sQ + wg * kWgTile + k * 32), tile_desc(sK + kb * kWgTile + k * 32), k > 0 ? 1u : 0u);
}
__device__ __forceinline__ void pack_afrag(uint32_t (&a)[4], const float (&x)[32], int kk) {
    a[0] = pack_bf16x2(x[8 * kk], x[8 * kk + 1]);
    a[1] = pack_bf16x2(x[8 * kk + 2], x[8 * kk + 3]);
    a[2] = pack_bf16x2(x[8 * kk + 4], x[8 * kk + 5]);
    a[3] = pack_bf16x2(x[8 * kk + 6], x[8 * kk + 7]);
}
// bf16 accumulator rows (r0, r0 + 8 of this lane) -> global [*, ld] (rows >= nrows skipped)
__device__ __forceinline__ void store_rows(bf16* base, long long ld, int r0, int nrows, const float (&x)[32], int t, float mul0, float mul1) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int col = 8 * j + 2 * t;
        if (r0 < nrows) *reinterpret_cast<uint32_t*>(base + static_cast<long long>(r0) * ld + col) = pack_bf16x2(x[4 * j] * mul0, x[4 * j + 1] * mul0);
        if (r0 + 8 < nrows)
            *reinterpret_cast<uint32_t*>(base + static_cast<long long>(r0 + 8) * ld + col) = pack_bf16x2(x[4 * j + 2] * mul1, x[4 * j + 3] * mul1);
    }
}
// accumulator rows -> one swizzled 64 x 64 bf16 tile in shared memory (the layout TMA writes and the descriptors read)
__device__ __forceinline__ void store_tile(uint32_t tile, int r, const float (&x)[32], int t) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        st_shared_u32(tile + swz(r, j) + 4 * t, pack_bf16x2(x[4 * j], x[4 * j + 1]));
        st_shared_u32(tile + swz(r + 8, j) + 4 * t, pack_bf16x2(x[4 * j + 2], x[4 * j + 3]));
    }
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
template <int NKB, bool VL = false>
__global__ void __launch_bounds__(NKB * 128, 1)
attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQKV, const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;   // 128B-swizzled tiles need 1 KB alignment
    uint8_t* smem = smem_raw + (base - raw);
    const uint32_t sQ = base, sK = base + NKB * kWgTile, sV = base + 2 * NKB * kWgTile;
    float* sbias = reinterpret_cast<float*>(smem + 3 * NKB * kWgTile);
    const uint32_t bar = base + 3 * NKB * kWgTile + NKB * kBlk * 4;
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int item = blockIdx.x, b = item / p.A, h = item % p.A;
    const unsigned bh = static_cast<unsigned>(item);
    const SeqSpan sp = seq_span<VL>(p, b, h);
    const int S = sp.len;                                 // rows of this sequence
    const int nkv = VL ? (S + kBlk - 1) / kBlk : NKB;     // its key blocks
    const int row0 = VL ? static_cast<int>(sp.row0) : b * S;
    if (VL && S == 0) return;                             // an empty sequence writes nothing

    if (tid == 0) {
        tma_prefetch_desc(&tmQKV);
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();
    if (tid == 0) {
        mbar_arrive_expect_tx(bar, 3 * nkv * kWgTile);
#pragma unroll
        for (int m = 0; m < 3; ++m)
#pragma unroll
            for (int kb = 0; kb < NKB; ++kb)
                if (!VL || kb < nkv) tma_load_2d(base + (m * NKB + kb) * kWgTile, &tmQKV, bar, m * p.H + h * kHd, row0 + kb * kBlk);
    }
    for (int i = tid; i < NKB * kBlk; i += NKB * 128) sbias[i] = key_bias2<VL>(p, b, i, S);
    const int q0 = wg * kBlk + warp * 16 + g;   // this lane's rows: q0, q0 + 8
    unsigned long long keep[NKB][2];
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb) {
        keep[kb][0] = keep_word(p, bh, q0, kb, NKB, t);
        keep[kb][1] = keep_word(p, bh, q0 + 8, kb, NKB, t);
    }
    __syncthreads();
    if (VL && wg >= nkv) return;   // query block past the sequence's end (warpgroup 0 stays and waits for the loads)
    mbar_wait(bar, 0);

    float s[NKB][32];
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb)
        if (!VL || kb < nkv) qk_block<NKB>(s[kb], sQ, sK, wg, kb);
    wgmma_commit();
    wgmma_wait<0>();

    // softmax of the two rows (a quad of lanes holds a row) in the exp2 domain
    const float sc2 = p.scale * kLog2e;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (VL && kb >= nkv) break;
            const float b0 = sbias[kb * kBlk + 8 * j + 2 * t], b1 = sbias[kb * kBlk + 8 * j + 2 * t + 1];
            s[kb][4 * j] = fmaf(s[kb][4 * j], sc2, b0); s[kb][4 * j + 1] = fmaf(s[kb][4 * j + 1], sc2, b1);
            s[kb][4 * j + 2] = fmaf(s[kb][4 * j + 2], sc2, b0); s[kb][4 * j + 3] = fmaf(s[kb][4 * j + 3], sc2, b1);
            mx[0] = fmaxf(mx[0], fmaxf(s[kb][4 * j], s[kb][4 * j + 1]));
            mx[1] = fmaxf(mx[1], fmaxf(s[kb][4 * j + 2], s[kb][4 * j + 3]));
        }
    float l[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                if (VL && kb >= nkv) break;
                const int r = c >> 1;
                float e = fast_ex2(s[kb][4 * j + c] - mx[r]);
                l[r] += e;
                // dropout: the 1/(1-p) factor is folded into the final normalisation
                if (!((keep[kb][r] >> (8 * j + (c & 1))) & 1ull)) e = 0.f;
                s[kb][4 * j + c] = e;
            }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    }

    // the A fragments must stay untouched until the MMAs reading them have retired: all of them are packed first
    uint32_t pa[NKB][4][4];
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
            if (!VL || kb < nkv) pack_afrag(pa[kb][kk], s[kb], kk);
    float o[32];
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
            if (!VL || kb < nkv)
                wgmma_m64n64k16_rs<1>(o, pa[kb][kk], tile_desc(sV + kb * kWgTile + kk * 2048), (kb > 0 || kk > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();

    const float dscale = p.drop_scale != 0.f ? p.drop_scale : 1.f;
    store_rows(p.ctx + (VL ? sp.row0 : static_cast<long long>(b) * S) * p.H + h * kHd, p.H, q0, S, o, t, dscale / l[0], dscale / l[1]);
    if (t == 0 && p.lse != nullptr) {
        float* lse = p.lse + (VL ? sp.stat0 : static_cast<long long>(item) * S);
        if (q0 < S) lse[q0] = (mx[0] + log2f(l[0])) * 0.6931471805599453f;
        if (q0 + 8 < S) lse[q0 + 8] = (mx[1] + log2f(l[1])) * 0.6931471805599453f;
    }
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
template <int NKB, bool VL = false>
__global__ void __launch_bounds__(NKB * 128, 1)
attn_bwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO, const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    const uint32_t sQ = base, sK = base + NKB * kWgTile, sV = base + 2 * NKB * kWgTile, sDO = base + 3 * NKB * kWgTile;
    const uint32_t sPS = base + 4 * NKB * kWgTile;   // [query block][key block] tiles of P_drop, later of dS
    float* sbias = reinterpret_cast<float*>(smem + (4 * NKB + NKB * NKB) * kWgTile);
    const uint32_t bar = base + (4 * NKB + NKB * NKB) * kWgTile + NKB * kBlk * 4;
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int item = blockIdx.x, b = item / p.A, h = item % p.A;
    const unsigned bh = static_cast<unsigned>(item);
    const long long ld = 3LL * p.H;
    const SeqSpan sp = seq_span<VL>(p, b, h);
    const int S = sp.len;
    const int nkv = VL ? (S + kBlk - 1) / kBlk : NKB;
    const int row0 = VL ? static_cast<int>(sp.row0) : b * S;
    const long long stat0 = VL ? sp.stat0 : static_cast<long long>(item) * S;
    if (VL && S == 0) return;
    // warpgroups whose 64-row block (of queries in pass 1 / 2, of keys for dV / dK) starts past the sequence's end issue no MMAs
    // but stay for the block-wide barriers
    const bool wg_live = !VL || wg < nkv;

    if (tid == 0) {
        tma_prefetch_desc(&tmQKV);
        tma_prefetch_desc(&tmDO);
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();
    if (tid == 0) {
        mbar_arrive_expect_tx(bar, 4 * nkv * kWgTile);
#pragma unroll
        for (int kb = 0; kb < NKB; ++kb) {
            if (VL && kb >= nkv) break;
#pragma unroll
            for (int m = 0; m < 3; ++m) tma_load_2d(base + (m * NKB + kb) * kWgTile, &tmQKV, bar, m * p.H + h * kHd, row0 + kb * kBlk);
            tma_load_2d(sDO + kb * kWgTile, &tmDO, bar, h * kHd, row0 + kb * kBlk);
        }
    }
    for (int i = tid; i < NKB * kBlk; i += NKB * 128) sbias[i] = key_bias2<VL>(p, b, i, S);
    const int r0 = warp * 16 + g;   // row of this lane inside its warpgroup's 64-row block (and r0 + 8)
    const int q0 = wg * kBlk + r0;
    float lse2[2], dr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int q = q0 + 8 * r;
        lse2[r] = q < S ? p.lse[stat0 + q] * kLog2e : INFINITY;   // +inf: probability 0
        dr[r] = q < S ? p.drow[stat0 + q] : 0.f;
    }
    unsigned long long keep[NKB][2];
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb) {
        keep[kb][0] = keep_word(p, bh, q0, kb, NKB, t);
        keep[kb][1] = keep_word(p, bh, q0 + 8, kb, NKB, t);
    }
    __syncthreads();
    mbar_wait(bar, 0);
    const float sc2 = p.scale * kLog2e;
    const float ds = p.drop_scale != 0.f ? p.drop_scale : 1.f;
    // probabilities of key block kb from raw scores (in place)
    auto probs = [&](float (&s)[32], int kb) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c)
                s[4 * j + c] = fast_ex2(fmaf(s[4 * j + c], sc2, sbias[kb * kBlk + 8 * j + 2 * t + (c & 1)]) - lse2[c >> 1]);
    };
    auto kept = [&](int kb, int j, int c) { return ((keep[kb][c >> 1] >> (8 * j + (c & 1))) & 1ull) != 0; };
    bf16* dqkv = p.dqkv + (VL ? sp.row0 : static_cast<long long>(b) * S) * ld + h * kHd;

    // ---- pass 1: P_drop -> shared memory; dV of this warpgroup's key block = P_drop^T dO ----
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb) {
        if (VL && (!wg_live || kb >= nkv)) break;
        float s[32];
        wgmma_fence();
        qk_block<NKB>(s, sQ, sK, wg, kb);
        wgmma_commit();
        wgmma_wait<0>();
        probs(s, kb);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c) s[4 * j + c] = kept(kb, j, c) ? s[4 * j + c] * ds : 0.f;
        store_tile(sPS + (wg * NKB + kb) * kWgTile, r0, s, t);
    }
    fence_proxy_async_smem();   // generic-proxy stores -> visible to the wgmma (async proxy) reads below
    __syncthreads();
    if (wg_live) {
        float acc[32];
        wgmma_fence();
#pragma unroll
        for (int qb = 0; qb < NKB; ++qb)
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                if (!VL || qb < nkv)
                    wgmma_m64n64k16_ss<1, 1>(acc, tile_desc(sPS + (qb * NKB + wg) * kWgTile + kk * 2048),
                                             tile_desc(sDO + qb * kWgTile + kk * 2048), (qb > 0 || kk > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        store_rows(dqkv + 2 * p.H, ld, q0, S, acc, t, 1.f, 1.f);   // rows of this warpgroup's block are keys here
    }
    __syncthreads();   // every read of the P_drop tiles is done: they are overwritten with dS below

    // ---- pass 2: dP = dO V^T, dS = P (dP_drop - D); dQ = dS K; dS -> shared memory; dK = dS^T Q ----
    float dq[32];
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb) {
        if (VL && (!wg_live || kb >= nkv)) break;
        float s[32], dp[32];
        wgmma_fence();
        qk_block<NKB>(s, sQ, sK, wg, kb);
#pragma unroll
        for (int k = 0; k < kHd / 16; ++k)
            wgmma_m64n64k16_ss<0, 0>(dp, tile_desc(sDO + wg * kWgTile + k * 32), tile_desc(sV + kb * kWgTile + k * 32), k > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        probs(s, kb);
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float dpd = kept(kb, j, c) ? dp[4 * j + c] * ds : 0.f;
                s[4 * j + c] *= dpd - dr[c >> 1];
            }
        store_tile(sPS + (wg * NKB + kb) * kWgTile, r0, s, t);
        uint32_t pa[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) pack_afrag(pa[kk], s, kk);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
            wgmma_m64n64k16_rs<1>(dq, pa[kk], tile_desc(sK + kb * kWgTile + kk * 2048), (kb > 0 || kk > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();   // the A fragments live in registers that the next block overwrites
    }
    if (wg_live) store_rows(dqkv, ld, q0, S, dq, t, p.scale, p.scale);
    fence_proxy_async_smem();
    __syncthreads();
    if (wg_live) {
        float acc[32];
        wgmma_fence();
#pragma unroll
        for (int qb = 0; qb < NKB; ++qb)
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                if (!VL || qb < nkv)
                    wgmma_m64n64k16_ss<1, 1>(acc, tile_desc(sPS + (qb * NKB + wg) * kWgTile + kk * 2048),
                                             tile_desc(sQ + qb * kWgTile + kk * 2048), (qb > 0 || kk > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        store_rows(dqkv + p.H, ld, q0, S, acc, t, p.scale, p.scale);
    }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
template <int NKB, bool VL = false>
static int launch_fwd_wgmma(const AttnParams& p, const CUtensorMap& tq, cudaStream_t st) {
    auto kern = attn_fwd_wgmma_kernel<NKB, VL>;
    static int configured[kMaxDevices] = {0};
    VB_CHECK_CUDA(ensure_dyn_smem(kern, AttnSmem<NKB>::FWD_BYTES, configured));
    ProfScope ps(st, PROF_ATTN_FWD, 4.0 * p.B * p.A * p.S * p.S * kHd, 1);
    VB_CHECK_CUDA(launch_pdl(kern, dim3(p.B * p.A), dim3(NKB * 128), AttnSmem<NKB>::FWD_BYTES, st, tq, p));
    return 0;
}
template <int NKB, bool VL = false>
static int launch_bwd_wgmma(const AttnParams& p, const CUtensorMap& tq, const CUtensorMap& td, cudaStream_t st) {
    auto kern = attn_bwd_wgmma_kernel<NKB, VL>;
    static int configured[kMaxDevices] = {0};
    VB_CHECK_CUDA(ensure_dyn_smem(kern, AttnSmem<NKB>::BWD_BYTES, configured));
    ProfScope ps(st, PROF_ATTN_DKV, 10.0 * p.B * p.A * p.S * p.S * kHd, 1);
    VB_CHECK_CUDA(launch_pdl(kern, dim3(p.B * p.A), dim3(NKB * 128), AttnSmem<NKB>::BWD_BYTES, st, tq, td, p));
    return 0;
}

int attn_fwd_wgmma(const AttnParams& p, const AttnDropOffset& off, cudaStream_t st) {
    const int nkb = (p.S + kBlk - 1) / kBlk;
    int rc = attn_keep_mask(p, off, nkb, st);
    if (rc) return rc;
    CUtensorMap tq;
    const bool vl = p.cu_seqlens != nullptr;
    const uint64_t rows = vl ? static_cast<uint64_t>(p.total) : static_cast<uint64_t>(p.B) * p.S;
    rc = make_tmap_bf16(&tq, p.qkv, 3ull * p.H, rows, 3ull * p.H, kBlk);
    if (rc) return rc;
    if (vl) {
        if (nkb == 1) rc = launch_fwd_wgmma<1, true>(p, tq, st);
        else if (nkb == 2) rc = launch_fwd_wgmma<2, true>(p, tq, st);
        else rc = launch_fwd_wgmma<3, true>(p, tq, st);
    } else if (nkb == 1) rc = launch_fwd_wgmma<1>(p, tq, st);
    else if (nkb == 2) rc = launch_fwd_wgmma<2>(p, tq, st);
    else rc = launch_fwd_wgmma<3>(p, tq, st);
    if (rc) return rc;
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int attn_bwd_wgmma(const AttnParams& p, cudaStream_t st, bool delta_ready) {
    const int nkb = (p.S + kBlk - 1) / kBlk;
    int rc = 0;
    if (!delta_ready) {
        rc = attn_delta(p, st);
        if (rc) return rc;
    }
    CUtensorMap tq, td;
    const bool vl = p.cu_seqlens != nullptr;
    const uint64_t rows = vl ? static_cast<uint64_t>(p.total) : static_cast<uint64_t>(p.B) * p.S;
    rc = make_tmap_bf16(&tq, p.qkv, 3ull * p.H, rows, 3ull * p.H, kBlk);
    if (rc) return rc;
    rc = make_tmap_bf16(&td, p.dctx, static_cast<uint64_t>(p.H), rows, static_cast<uint64_t>(p.H), kBlk);
    if (rc) return rc;
    if (vl) {
        if (nkb == 1) rc = launch_bwd_wgmma<1, true>(p, tq, td, st);
        else if (nkb == 2) rc = launch_bwd_wgmma<2, true>(p, tq, td, st);
        else rc = launch_bwd_wgmma<3, true>(p, tq, td, st);
    } else if (nkb == 1) rc = launch_bwd_wgmma<1>(p, tq, td, st);
    else if (nkb == 2) rc = launch_bwd_wgmma<2>(p, tq, td, st);
    else rc = launch_bwd_wgmma<3>(p, tq, td, st);
    if (rc) return rc;
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace vb
