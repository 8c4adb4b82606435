// vb_attention.cuh — device helpers shared by the attention kernels. The sequence length alone picks the kernels
// (attn_route, vb_internal.h): vb_attention_wgmma.cu: wgmma / TMA kernels for seq <= 192; vb_attention_head.cu:
// persistent whole-head mma.sync kernels for 192 < seq <= 256; vb_attention.cu: staged kernels for seq > 256.
#pragma once

#include "../../include/vbert_b200.h"
#include "vb_common.cuh"

namespace vb {


constexpr int kHd = 64;             // head dim
constexpr int kBlk = 64;            // rows per tile (queries or keys)
constexpr int kTileBytes = kBlk * kHd * 2;
constexpr float kLog2e = 1.4426950408889634f;

struct AttnParams {
    const bf16* qkv;   // [B*S, 3H]
    const float* mask_bias;  // [B, S] additive key bias, natural-log domain ((1-mask) * -10000)
    bf16* ctx;         // [B*S, H]        (fwd out / bwd: O)
    float* lse;        // [B, A, S]       natural-log domain
    const bf16* dctx;  // [B*S, H]        (bwd)
    bf16* dqkv;        // [B*S, 3H]       (bwd out)
    float* drow;       // [B, A, S]       (bwd scratch: rowsum(dO * O))
    unsigned long long* keep;  // [B*A, nkb*64 rows, nkb] 64-bit keep-masks (bit = key within the 64-key block); dropout only
    int B, S, A, H;
    float scale;       // 1/sqrt(head_dim)
    float drop_scale;  // 1/(1-p) or 0
    unsigned drop_thresh16;  // attention: 8-bit threshold, round(p * 256)
    unsigned drop_seed;     // attn_seed_fold(seed, stream id) of the call
    // variable-length ("unpadded") calls: sequence b owns the packed rows [cu_seqlens[b], cu_seqlens[b+1]) of `total`; S is then
    // the longest sequence (it sizes the grid and the keep-mask layout), lse / drow are [A, total], and mask_bias is unused
    const int* cu_seqlens;  // device [B + 1]; nullptr for dense calls
    int total;
};

// The rows one (sequence b, head h) works on: the first packed row, the sequence length and the base of its lse / drow
// entries. Dense: (b S, S, (b A + h) S). Varlen: (cu[b], len_b, h total + cu[b]), with the table clamped so that a bad
// cu_seqlens cannot send a kernel outside [0, total) rows or past S rows per sequence.
struct SeqSpan {
    long long row0;
    int len;
    long long stat0;
};
template <bool VL>
__device__ __forceinline__ SeqSpan seq_span(const AttnParams& p, int b, int h) {
    SeqSpan s;
    if constexpr (VL) {
        int lo = __ldg(p.cu_seqlens + b), hi = __ldg(p.cu_seqlens + b + 1);
        lo = min(max(lo, 0), p.total);
        hi = min(max(hi, lo), p.total);
        s.row0 = lo;
        s.len = min(hi - lo, p.S);
        s.stat0 = static_cast<long long>(h) * p.total + lo;
    } else {
        s.row0 = static_cast<long long>(b) * p.S;
        s.len = p.S;
        s.stat0 = (static_cast<long long>(b) * p.A + h) * p.S;
    }
    return s;
}
// additive key bias in the exp2 domain: the caller's mask when dense; every key of the sequence is valid when varlen
template <bool VL>
__device__ __forceinline__ float key_bias2(const AttnParams& p, int b, int key, int len) {
    if constexpr (VL) return key < len ? 0.f : -INFINITY;
    else return key < p.S ? p.mask_bias[static_cast<long long>(b) * p.S + key] * kLog2e : -INFINITY;
}

// vb_set_dropout_offset: a forward call whose offset is set draws its keep bits with attn_seed_fold(seed + *offset, stream_id)
// instead of p.drop_seed, in the *_off kernels (the backward kernels read the bits the forward stored and need no seed)
struct AttnDropOffset {
    const unsigned long long* offset;   // nullptr: unset, or no dropout
    unsigned long long seed;
    unsigned stream_id;
};
// The 32-bit seed of the attention keep-bit hash: the per-layer stream id folded into the 64-bit seed (splitmix64 finaliser).
// On the host for a call with its seed by value, on the device when the seed offset lives in device memory.
__host__ __device__ __forceinline__ unsigned attn_seed_fold(unsigned long long seed, unsigned stream_id) {
    unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (stream_id + 1ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return static_cast<unsigned>(z ^ (z >> 31));
}

// ------------------------------------------------------------------------------------------------
// small device helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t swz(int row, int chunk) {  // byte offset inside a 64x64 bf16 tile
    return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;  // src-size 0 => zero fill
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// 64 x 64 bf16 tile: rows row0..row0+63 of a [*, ld] matrix starting at column col0; rows >= nrows -> 0
template <int NT = 128>
__device__ __forceinline__ void load_tile(uint32_t tile, const bf16* base, long long ld, int row0, int nrows,
                                          int tid) {
#pragma unroll
    for (int i = 0; i < 512 / NT; ++i) {
        const int idx = tid + i * NT;
        const int r = idx >> 3, c = idx & 7;
        const bool ok = (row0 + r) < nrows;
        const bf16* src = base + static_cast<long long>(ok ? row0 + r : 0) * ld + c * 8;
        cp_async16(tile + swz(r, c), src, ok);
    }
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A fragments (16 rows x 64 k) of rows r0..r0+15 of a swizzled [64][64] tile
__device__ __forceinline__ void load_afrag(uint32_t (&a)[4][4], uint32_t tile, int r0, int lane) {
    const int row = r0 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        const int chunk = ks * 2 + (lane >> 4);
        ldsm_x4(tile + swz(row, chunk), a[ks][0], a[ks][1], a[ks][2], a[ks][3]);
    }
}
// acc(16 x 64 n) += A(16 x 64 k) * T^T, T = tile [n=64][k=64] row-major; only the first `nvalid`
// rows of T (n index) carry data — whole 16-wide n pairs beyond it are skipped (warp-uniform).
__device__ __forceinline__ void gemm_nt(float (&acc)[8][4], const uint32_t (&a)[4][4], uint32_t tile, int lane,
                                        int nvalid = 64) {
    // k-step outermost: consecutive MMAs hit different accumulators (no back-to-back dependent HMMA)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {
            if (np * 16 < nvalid) {
                const int row = np * 16 + (lane & 7) + (lane >> 4) * 8;
                const int chunk = ks * 2 + ((lane >> 3) & 1);
                uint32_t b0, b1, b2, b3;
                ldsm_x4(tile + swz(row, chunk), b0, b1, b2, b3);
                mma16816(acc[2 * np], a[ks], b0, b1);
                mma16816(acc[2 * np + 1], a[ks], b2, b3);
            }
        }
    }
}
// acc(16 x 64 n) += A(16 x 64 k) * T, T = tile [k=64][n=64] row-major; k-steps beyond `kvalid` rows
// of T are skipped (their A columns are exact zeros).
__device__ __forceinline__ void gemm_nn(float (&acc)[8][4], const uint32_t (&a)[4][4], uint32_t tile, int lane,
                                        int kvalid = 64) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        if (ks * 16 < kvalid) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                const int row = ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                const int chunk = np * 2 + (lane >> 4);
                uint32_t b0, b1, b2, b3;
                ldsm_x4_t(tile + swz(row, chunk), b0, b1, b2, b3);
                mma16816(acc[2 * np], a[ks], b0, b1);
                mma16816(acc[2 * np + 1], a[ks], b2, b3);
            }
        }
    }
}
// MT m-tiles per warp (16*MT rows): every B fragment fetched by ldmatrix feeds 2*MT MMAs
template <int MT>
__device__ __forceinline__ void gemm_nt_mt(float (&acc)[MT][8][4], const uint32_t (&a)[MT][4][4], uint32_t tile, int lane,
                                           int nvalid) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {
            if (np * 16 < nvalid) {
                const int row = np * 16 + (lane & 7) + (lane >> 4) * 8;
                const int chunk = ks * 2 + ((lane >> 3) & 1);
                uint32_t b0, b1, b2, b3;
                ldsm_x4(tile + swz(row, chunk), b0, b1, b2, b3);
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    mma16816(acc[mt][2 * np], a[mt][ks], b0, b1);
                    mma16816(acc[mt][2 * np + 1], a[mt][ks], b2, b3);
                }
            }
        }
    }
}
template <int MT>
__device__ __forceinline__ void gemm_nn_mt(float (&acc)[MT][8][4], const uint32_t (&a)[MT][4][4], uint32_t tile, int lane,
                                           int kvalid) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        if (ks * 16 < kvalid) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                const int row = ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                const int chunk = np * 2 + (lane >> 4);
                uint32_t b0, b1, b2, b3;
                ldsm_x4_t(tile + swz(row, chunk), b0, b1, b2, b3);
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    mma16816(acc[mt][2 * np], a[mt][ks], b0, b1);
                    mma16816(acc[mt][2 * np + 1], a[mt][ks], b2, b3);
                }
            }
        }
    }
}
// half-width variant: acc(16 x 32) = A * T^T for n in [32*half, 32*half + 32)
__device__ __forceinline__ void gemm_nt_half(float (&acc)[4][4], const uint32_t (&a)[4][4], uint32_t tile, int lane,
                                             int half, int nvalid) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int np = half * 2 + q;
            if (np * 16 < nvalid) {
                const int row = np * 16 + (lane & 7) + (lane >> 4) * 8;
                const int chunk = ks * 2 + ((lane >> 3) & 1);
                uint32_t b0, b1, b2, b3;
                ldsm_x4(tile + swz(row, chunk), b0, b1, b2, b3);
                mma16816(acc[2 * q], a[ks], b0, b1);
                mma16816(acc[2 * q + 1], a[ks], b2, b3);
            }
        }
    }
}
__device__ __forceinline__ void cp_async_wait_dyn(int pending) {  // allow `pending` newest groups in flight
    switch (pending) {
        case 0: cp_async_wait<0>(); break;
        case 1: cp_async_wait<1>(); break;
        case 2: cp_async_wait<2>(); break;
        default: cp_async_wait<3>(); break;
    }
}
// accumulator tile (16 x 64, fp32) -> A fragments (bf16) for the next GEMM
__device__ __forceinline__ void acc_to_afrag(uint32_t (&a)[4][4], const float (&p)[8][4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        a[j][0] = pack_bf16x2(p[2 * j][0], p[2 * j][1]);
        a[j][1] = pack_bf16x2(p[2 * j][2], p[2 * j][3]);
        a[j][2] = pack_bf16x2(p[2 * j + 1][0], p[2 * j + 1][1]);
        a[j][3] = pack_bf16x2(p[2 * j + 1][2], p[2 * j + 1][3]);
    }
}
__device__ __forceinline__ void zero_acc(float (&c)[8][4]) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) c[i][j] = 0.f;
}
// Attention-probability dropout (reference modeling.py:251). The keep decisions are drawn ONCE, in the forward
// kernel (counter hash of (batch*head, query row, key block, lane quad) -> 4 x 8 random bits per hash), applied
// there, and written out as a packed bit-mask: one 64-bit word per (query row, 64-key block). Both backward
// kernels read the bits back instead of re-hashing — the kernels are instruction-issue bound and the per-element
// hashing was ~45 % of their instruction count. The drop probability is quantised to round(p*256)/256
// (0.1 -> 26/256) and survivors are scaled by 256/(256 - that), so E[dropout(P)] = P exactly.
// attn_keep16 (staged kernels): for one query row, the 16 elements a thread owns in a 64-key block (keys nt*8 + 2t + {0,1}).
// Hash counters: 16 w + 4 t + j (j < 4), where w = (bh * nkb*64 + q) * nkb + kb is the index of the 64-bit keep word of
// (query row q, key block kb) in the mask buffer. Every (bh, q, kb, t, j) with q < nkb*64 therefore gets its own counter, as
// long as B*A * nkb*64 * nkb * 16 < 2^32 (checked on the host), and no two keep words of a call share a random bit.
__device__ __forceinline__ uint32_t attn_keep16(unsigned seed, unsigned bh, int q, int kb, int t, int nkb, unsigned thresh8) {
    const unsigned np64 = static_cast<unsigned>(nkb) * kBlk;
    const unsigned w = (bh * np64 + static_cast<unsigned>(q)) * static_cast<unsigned>(nkb) + static_cast<unsigned>(kb);
    const unsigned base = (w << 4) + (static_cast<unsigned>(t) << 2);
    uint32_t bits = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {  // hash j covers n-tiles 2j and 2j+1
        const uint32_t h = mix32((base + j) ^ seed);
        bits |= static_cast<uint32_t>((h & 0xffu) >= thresh8) << (4 * j);
        bits |= static_cast<uint32_t>(((h >> 8) & 0xffu) >= thresh8) << (4 * j + 1);
        bits |= static_cast<uint32_t>(((h >> 16) & 0xffu) >= thresh8) << (4 * j + 2);
        bits |= static_cast<uint32_t>((h >> 24) >= thresh8) << (4 * j + 3);
    }
    return bits;  // bit (2*nt + c) = keep of key nt*8 + 2t + c
}
// spread a thread's 16 keep bits to their key positions inside the 64-bit block mask and OR over the quad
__device__ __forceinline__ unsigned long long quad_mask64(uint32_t bits16, int t) {
    unsigned long long m = 0;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) m |= static_cast<unsigned long long>((bits16 >> (2 * nt)) & 3u) << (nt * 8 + 2 * t);
    m |= __shfl_xor_sync(0xffffffffu, m, 1);
    m |= __shfl_xor_sync(0xffffffffu, m, 2);
    return m;
}
// store a 16 x 64 accumulator tile as bf16 rows of a [*, ld] matrix (rows >= nrows skipped)
__device__ __forceinline__ void store_acc(bf16* base, long long ld, int row0, int nrows, const float (&c)[8][4],
                                          int lane, float mul0, float mul1) {
    const int g = lane >> 2, t = lane & 3;
    const int ra = row0 + g, rb = row0 + g + 8;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        const int col = nt * 8 + 2 * t;
        if (ra < nrows)
            *reinterpret_cast<uint32_t*>(base + static_cast<long long>(ra) * ld + col) =
                pack_bf16x2(c[nt][0] * mul0, c[nt][1] * mul0);
        if (rb < nrows)
            *reinterpret_cast<uint32_t*>(base + static_cast<long long>(rb) * ld + col) =
                pack_bf16x2(c[nt][2] * mul1, c[nt][3] * mul1);
    }
}


constexpr int kMaxSub = 4;  // 64-row tiles per resident stage

// The forward launchers of the two fused routes draw the dropout keep bits (attn_keep_mask) before their kernel.
// delta_ready: p.drow already holds D = rowsum(dO * O) (written by the epilogue of the GEMM that produced dO,
// vb_gemm_args.delta_out); otherwise the backward launchers run attn_delta first.
// Every launcher serves dense calls and, when p.cu_seqlens != nullptr, variable-length ones (a separate instantiation of each
// kernel, so the dense code is unchanged).
// whole-head persistent kernels (vb_attention_head.cu), 192 < seq <= 256; nkb = ceil(S / 64)
int attn_fwd_head(const AttnParams& p, const AttnDropOffset& off, int nkb, cudaStream_t st);
int attn_bwd_head(const AttnParams& p, int nkb, cudaStream_t st, bool delta_ready);
int attn_keep_mask(const AttnParams& p, const AttnDropOffset& off, int nkb, cudaStream_t st);
int attn_delta(const AttnParams& p, cudaStream_t st);
// wgmma / TMA / mbarrier kernels (vb_attention_wgmma.cu), seq <= 192
int attn_fwd_wgmma(const AttnParams& p, const AttnDropOffset& off, cudaStream_t st);
int attn_bwd_wgmma(const AttnParams& p, cudaStream_t st, bool delta_ready);
int make_tmap_bf16(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld_elems, uint32_t box_outer);

}  // namespace vb
