// vb_internal.h — declarations shared between the translation units of libvbert_b200 (not part of the ABI).
#pragma once
#include "../../include/vbert_b200.h"
#include "vb_common.cuh"

namespace vb {

int gemm(const vb_gemm_args& a, cudaStream_t st);
bool gemm_gp_tiled_ok(int M, int N);
bool gemm_delta_ok(int M, int N);
int ln_fwd(const void* x, long long ldx, const float* gamma, const float* beta, void* y, long long ldy, float* mean,
           float* rstd, int rows, int H, float eps, cudaStream_t st);
int ln_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const float* gamma, void* dx,
           void* dx_drop, float* dgamma, float* dbeta, float* dbias, int rows, int H, float dropout_p,
           unsigned long long seed, unsigned stream_id, float in_dropout_p, unsigned in_stream_id, cudaStream_t st,
           bool rows_only = false);   // rows_only: dgamma, dbeta and dbias are all NULL and no column reduction runs
// The attention kernels that serve a call, from its sequence length (varlen calls: the longest one): the wgmma kernels up to
// 192 (their backward keeps Q, K, V, dO and P/dS of the whole head in shared memory), the whole-head mma.sync kernels up to
// 256, the staged kernels beyond. The two fused routes take a pre-computed D = rowsum(dO * O) (delta_ready below).
enum class AttnRoute { Wgmma, Head, Staged };
inline AttnRoute attn_route(int S) { return S <= 192 ? AttnRoute::Wgmma : S <= 256 ? AttnRoute::Head : AttnRoute::Staged; }
int attn_fwd(const void* qkv, const float* mask_bias, void* ctx, float* lse, void* keep, int B, int S, int A, int H,
             float dropout_p, unsigned long long seed, unsigned stream_id, cudaStream_t st);
int attn_bwd(const void* qkv, const float* mask_bias, const void* ctx, const float* lse, const void* keep,
             const void* dctx, void* dqkv, float* drow, int B, int S, int A, int H, float dropout_p,
             unsigned long long seed, unsigned stream_id, cudaStream_t st, bool delta_ready = false);
// variable-length attention: sequence b owns packed rows [cu_seqlens[b], cu_seqlens[b+1]) (device), at most max_seq of them;
// lse / drow are [A, total]; need_lse = false (a forward no backward follows) lets lse be NULL, as the dense call always does
int attn_fwd_varlen(const void* qkv, const int* cu_seqlens, void* ctx, float* lse, void* keep, int B, int max_seq, int total,
                    int A, int H, float dropout_p, unsigned long long seed, unsigned stream_id, cudaStream_t st, bool need_lse = true);
int attn_bwd_varlen(const void* qkv, const int* cu_seqlens, const void* ctx, const float* lse, const void* keep,
                    const void* dctx, void* dqkv, float* drow, int B, int max_seq, int total, int A, int H, float dropout_p,
                    unsigned long long seed, unsigned stream_id, cudaStream_t st, bool delta_ready = false);
long long attn_keep_bytes(int B, int S, int A);
// the pre-dropout attention maps softmax(QK^T / 8 + mask_bias) of a dense call, fp32 [B, A, S, S] (vb_attention_probs.cu)
int attn_probs(const void* qkv, const float* mask_bias, float* probs, int B, int S, int A, int H, cudaStream_t st);
// deterministic mode (vb_set_deterministic; see vb_common.cuh det_ws)
int wgrad_splits(long long tiles, int k_blocks);   // split-K factor of an fp32 output (vb_gemm.cu)
long long gemm_tiles(int M, int N);
int gemm_k_blocks(int K);
long long ln_bwd_det_bytes(int rows, int H);       // workspace of one ln_bwd call in deterministic mode
long long colsum_det_bytes(int M, int N);          // ... of one colsum call
long long embed_bwd_det_bytes(int B, int T, int V, int H, long long sort_temp);   // ... of embed_bwd (sort_temp < 0: a bound)
long long embed_sort_temp_bytes(int B, int T, int V);
int partials_reduce(const float* part, int parts, int width, int seg, float* o0, float* o1, float* o2, cudaStream_t st);
int colsum(const void* x, long long ld, float* out, int M, int N, cudaStream_t st);
int cast_f32_bf16(const float* src, void* dst, long long n, cudaStream_t st);
int cast_bf16_f32(const void* src, float* dst, long long n, cudaStream_t st);
int mask_bias(const long long* input_mask, const long long* image_mask, float* out, int B, int T, int V, cudaStream_t st);

struct EmbedParams {
    const long long* ids; const long long* tt; const long long* vt;
    const bf16* vis_proj;
    const float* word; const float* pos; const float* type; const float* pos_vis; const float* type_vis;
    const float* gamma; const float* beta;
    bf16* pre; bf16* y; float* mean; float* rstd;
    int B, T, V, H, vocab, max_pos, n_types;
    float eps;
    float drop_scale; unsigned drop_thresh16; unsigned long long drop_seed; unsigned drop_stream;
    const unsigned long long* drop_offset;   // non-null: the dropout seed is drop_seed + *drop_offset (vb_set_dropout_offset)
};
struct EmbedBwdParams {
    const bf16* de;
    const long long* ids; const long long* tt; const long long* vt;
    float* dword; float* dpos; float* dtype; float* dpos_vis; float* dtype_vis;
    bf16* dvis;
    int B, T, V, H, vocab, max_pos, n_types;
};
int embed_fwd(const EmbedParams& p, cudaStream_t st);
int embed_bwd(const EmbedBwdParams& p, cudaStream_t st);


}  // namespace vb
