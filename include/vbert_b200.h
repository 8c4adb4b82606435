/*
 * vbert_b200.h — C ABI of libvbert_b200.so: the VisualBERT encoder hot path as sm_90a (H100) kernels.
 *
 * Drop-in boundary (SURVEY.md §8b): every entry point takes plain device pointers, sizes and a
 * cudaStream_t (passed as void*); no torch types, no allocation of persistent state, re-entrant.
 * All functions return 0 on success, non-zero on error; vb_last_error() returns the message of the
 * last failure on the calling thread. The library never throws and never calls exit().
 *
 * Each entry point names the reference code it replaces
 * (paths under uclanlp/visualbert: visualbert/pytorch_pretrained_bert/modeling.py = "M.py").
 *
 * Layout conventions: activations are row-major [rows = batch*seq, features], bf16 (2 bytes);
 * parameters handed to the library are bf16 copies ("compute weights") of the fp32 master
 * parameters in nn.Linear layout [out, in]; statistics, biases, LayerNorm affine and all
 * parameter gradients are fp32.
 */
#ifndef VBERT_B200_H
#define VBERT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VB_ABI_VERSION 4

/* ---- library ---------------------------------------------------------------------------- */
int vb_abi_version(void);
const char* vb_last_error(void);
/* number of kernel launches issued by this library on the calling process since load */
int64_t vb_launch_count(void);
/* Live profiling: when enabled every launcher brackets its kernels with CUDA events on the launch stream.
 * vb_profile_read synchronises the device and returns, per category, the summed kernel time [ms], the
 * algorithmic work (FLOPs for the tensor-core kernels, bytes for the HBM-bound ones) and the number of launches
 * since the previous read; arrays of VB_PROFILE_CATEGORIES entries:
 * 0 gemm fwd, 1 gemm dgrad, 2 gemm wgrad (all gemm_wgmma_kernel), 3 attention fwd, 4 attention dQ,
 * 5 attention dK/dV, 6 layernorm fwd, 7 layernorm bwd, 8 column sums, 9 embedding, 10 other. */
#define VB_PROFILE_CATEGORIES 11
void vb_profile_enable(int on);
int vb_profile_read(double* ms, double* work, int64_t* launches);

/* Deterministic reductions (torch.use_deterministic_algorithms). While a workspace is set ON THE CALLING THREAD, every entry
 * point that reduces across CTAs does so in a fixed order: split-K weight gradients, LayerNorm dgamma/dbeta/dbias, column sums,
 * embedding-table gradients, the BertAdam gradient norms. Results are then bitwise reproducible for the same inputs, shapes,
 * build and GPU model. workspace = NULL turns it off (the default: today's kernels, unchanged). The library allocates nothing;
 * a call that needs more scratch than `bytes` fails with vb_last_error() naming the bytes it needs, BEFORE launching anything
 * (a split-K GEMM whose slabs do not fit lowers its split factor instead). The workspace must be 256-byte aligned.
 * The workspace is used in stream order: do not share one workspace between streams that run concurrently. */
int vb_set_deterministic(void* workspace, int64_t bytes);
/* bytes of workspace that every call of an encoder / embedding / MLM-decoder / BertAdam of this shape needs
 * (rows = the largest M of any call; adam_chunks = n_chunks of the largest vb_bert_adam_step). Arguments that do not apply may
 * be 0 (e.g. inter and vocab for a BertAdam-only workspace); for the embedding pass inter = visual_dim. -1 on a bad shape. */
int64_t vb_deterministic_workspace_bytes(int64_t rows, int32_t hidden, int32_t inter, int32_t vocab, int32_t adam_chunks);

/* Dropout seed offset in device memory (CUDA graphs). While `offset` is set ON THE CALLING THREAD, every dropout a call draws or
 * regenerates — GEMM epilogues, LayerNorm backward (hidden dropout and in_dropout), embeddings, attention keep bits — uses the seed
 * (seed argument or descriptor seed) + *offset (mod 2^64): the bits equal those of the same call with that sum passed by value.
 * offset points at one uint64 in DEVICE memory (8-byte aligned); the kernels read it when they run, the host never does, so a
 * captured graph that is replayed after the value changed draws fresh bits. Calls without dropout are unaffected. offset = NULL
 * turns it off (the default: the same kernels, grids and bits as without this call). Launches issued while their stream is
 * capturing skip the vb_profile_enable event pairs; nothing else in the library synchronises with the host or allocates. */
int vb_set_dropout_offset(const uint64_t* offset);

/* ---- GEMM core (wgmma + TMA + mbarrier) --------------------------------------------------- */
/* epilogue selectors */
#define VB_EPI_NONE 0
#define VB_EPI_GELU 1  /* u = acc + bias: aux_out = gelu(u), D = gelu'(u)   — M.py:56-61, 302-305 */
#define VB_EPI_DGELU 2 /* D = acc * aux_in  (aux_in = the gelu'(u) saved by VB_EPI_GELU) — backward of M.py:304 */
/* 3 is retired and refused as unknown */
#define VB_EPI_GELU_FWD 4 /* u = acc + bias: D = gelu(u) and nothing else (no aux_out, no aux_in, no gp_tiled) — the FFN-up GEMM of a
                           * forward that no backward follows (evaluation under torch.no_grad(), train.py:292-325). D holds bit for
                           * bit what VB_EPI_GELU writes to aux_out; K-major A and B and a bf16 D only. */
/* The GELU epilogues take no dropout and no addend: vb_gemm refuses such a call. */

typedef struct {
    /* D[M,N] = epilogue( sum_k A(m,k) * B(n,k) )
     * a_mn_major = 0: A stored [M,K] row-major (K contiguous), lda = row stride (elements)
     * a_mn_major = 1: A stored [K,M] row-major (M contiguous)  — used for weight gradients
     * b_mn_major = 0: B stored [N,K] row-major (nn.Linear weight layout for y = x W^T)
     * b_mn_major = 1: B stored [K,N] row-major                  — used for input gradients */
    const void* A; int64_t lda; int32_t a_mn_major;
    const void* B; int64_t ldb; int32_t b_mn_major;
    int32_t M, N, K;
    void* D; int64_t ldd;
    int32_t d_fp32;   /* 0: D is bf16; 1: D is fp32 and the result is ACCUMULATED into D (red.add) */
    int32_t splits;   /* unused: the split-K factor of a d_fp32 output is chosen from the shape (field kept for the ABI) */
    const float* bias;            /* fp32 [N] or NULL */
    const void* addend; int64_t ld_add; /* bf16 [M,N] added after bias/dropout (residual) or NULL */
    int32_t epilogue;             /* VB_EPI_* */
    const void* aux_in;           /* VB_EPI_DGELU: gelu'(u), bf16 [M,N] */
    void* aux_out;                /* VB_EPI_GELU: gelu(u), bf16 [M,N] */
    int64_t ld_aux;
    /* inverted dropout on (acc + bias) before the addend — M.py:272, 317 (nn.Dropout) */
    float dropout_p; uint64_t dropout_seed; uint32_t dropout_stream;
    /* gp_tiled = 1 (VB_EPI_GELU / VB_EPI_DGELU only, and only when vb_gemm_gp_tiled_ok(M, N)): gelu'(u) — D of the GELU
     * epilogue, aux_in of the DGELU epilogue — is kept in the library's TILE-NATIVE order instead of row-major [M, N]:
     * same M * N bf16 elements; for the 256 x 256 tile (mb, nb), CTA rank r (rows 128 r ..), epilogue warp w = 4 * column-half +
     * row-quarter, 16-column chunk k, lane l: the 16 elements of row 256 mb + 128 r + 32 (w % 4) + l, columns
     * 256 nb + 128 (w / 4) + 16 k .. + 15 sit at element ((((mb * N/256 + nb) * 2 + r) * 8 + w) * 8 + k) * 512 + 16 l.
     * The tensor has exactly one producer and one consumer — two GEMM epilogues in which the same thread owns the same
     * 16 columns — so both touch whole 1 KB warp blocks instead of 32-byte pieces of 32 rows. vb_layer_fwd / _bwd use it
     * for vb_layer_acts.u whenever the shape allows. */
    int32_t gp_tiled;
    /* delta_out != NULL (bf16 output, b_mn_major = 1, no bias / addend / dropout / epilogue; vb_gemm_delta_ok(M, N)): besides D
     * the call writes delta_out[b][h][s] = sum_{d < 64} D[b * delta_seq + s][64 h + d] * delta_ctx[same element]
     * (fp32 [M / delta_seq][N / 64][delta_seq]; delta_ctx bf16 [M, N] row-major) — the D = rowsum(dO * O) term of the attention
     * backward, computed in the epilogue of the GEMM that produces dO (input gradient of attention.output.dense), where one
     * thread holds two whole heads of a row. vb_layer_bwd uses it to drop the separate pass over dO and O. */
    const void* delta_ctx; float* delta_out; int32_t delta_seq;
} vb_gemm_args;
int vb_gemm_delta_ok(int32_t M, int32_t N);
/* 1 when gp_tiled is supported for this output shape on this build (M, N multiples of 256, CTA-pair kernels enabled) */
int vb_gemm_gp_tiled_ok(int32_t M, int32_t N);

int vb_gemm(const vb_gemm_args* args, void* stream);

/* ---- BertLayerNorm (M.py:162-175) -------------------------------------------------------- */
/* y = gamma * (x - mean) / sqrt(var + eps) + beta over the last dim; x, y bf16 [rows, hidden] with row strides ldx, ldy;
 * mean / rstd (fp32 [rows]) are written when non-NULL (saved for backward).
 * The kernels move rows in 16-byte pieces: x, y, gamma and beta must be 16-byte aligned and ldx, ldy multiples of 8 that are
 * >= hidden; in the backward dy, x, gamma, dx and dx_drop must be 16-byte aligned. A call that breaks this returns an error. */
int vb_layernorm_fwd(const void* x, int64_t ldx, const float* gamma, const float* beta, void* y, int64_t ldy,
                     float* mean, float* rstd, int32_t rows, int32_t hidden, float eps, void* stream);
/* dx = LN'(dy); dgamma/dbeta/dbias (fp32 [hidden]) are ACCUMULATED; dbias = column sum of the
 * gradient entering the Linear in front of the LayerNorm. With dropout_p > 0, dx_drop receives
 * dx * keep/(1-p) (gradient through the hidden dropout of M.py:272/317) and dbias sums dx_drop.
 * in_dropout_p > 0 re-applies the keep mask of a dropout that FOLLOWED the LayerNorm (M.py:1256). */
int vb_layernorm_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const float* gamma,
                     void* dx, void* dx_drop, float* dgamma, float* dbeta, float* dbias, int32_t rows,
                     int32_t hidden, float dropout_p, uint64_t dropout_seed, uint32_t dropout_stream,
                     float in_dropout_p, uint32_t in_dropout_stream, void* stream);

/* ---- BertSelfAttention core (M.py:241-256) ----------------------------------------------- */
/* qkv bf16 [batch*seq, 3*hidden] (Q | K | V), mask_bias fp32 [batch, seq] additive key bias,
 * ctx bf16 [batch*seq, hidden], lse fp32 [batch, heads, seq]. head_dim must be 64. qkv, and in the backward ctx and dctx,
 * must be 16-byte aligned (the kernels load them in 16-byte pieces); a call with one that is not returns an error.
 * keep_mask: vb_attention_keep_bytes(batch, seq, heads) bytes, written by forward and read by backward when
 * dropout_p > 0 (packed keep bits of the attention-probability dropout, M.py:251); may be NULL otherwise. */
int64_t vb_attention_keep_bytes(int32_t batch, int32_t seq, int32_t heads);
int vb_attention_fwd(const void* qkv, const float* mask_bias, void* ctx, float* lse, void* keep_mask, int32_t batch,
                     int32_t seq, int32_t heads, int32_t hidden, float dropout_p, uint64_t dropout_seed,
                     uint32_t dropout_stream, void* stream);
/* dqkv bf16 [batch*seq, 3*hidden] out; drow fp32 [batch, heads, seq] scratch. */
int vb_attention_bwd(const void* qkv, const float* mask_bias, const void* ctx, const float* lse, const void* keep_mask,
                     const void* dctx, void* dqkv, float* drow, int32_t batch, int32_t seq, int32_t heads,
                     int32_t hidden, float dropout_p, uint64_t dropout_seed, uint32_t dropout_stream, void* stream);
/* Variable-length ("unpadded") attention: `batch` sequences packed without padding. qkv bf16 [total, 3*hidden], sequence b
 * owns rows [cu_seqlens[b], cu_seqlens[b+1]); cu_seqlens is int32 [batch + 1] in DEVICE memory; max_seq >= every length.
 * ctx bf16 [total, hidden], dqkv bf16 [total, 3*hidden], lse and drow fp32 [heads, total]; keep_mask as for the dense call
 * with seq = max_seq (vb_attention_keep_bytes(batch, max_seq, heads)). There is no mask: every row of a sequence is a valid
 * key. Only rows inside [cu[b], cu[b] + len_b) are written. The route (wgmma / whole-head / staged) is chosen from
 * max_seq as the dense call chooses it from seq. The alignment rule of the dense call applies.
 * Caller contract (not checked, that would need a host synchronisation): cu_seqlens is non-decreasing from 0 to at most total
 * and no length exceeds max_seq. The kernels clamp every length to [0, max_seq] and every row range to [0, total), so a bad
 * table gives wrong values but no access outside the tensors. */
int vb_attention_fwd_varlen(const void* qkv, const int32_t* cu_seqlens, void* ctx, float* lse, void* keep_mask, int32_t batch,
                            int32_t max_seq, int32_t total, int32_t heads, int32_t hidden, float dropout_p, uint64_t dropout_seed,
                            uint32_t dropout_stream, void* stream);
int vb_attention_bwd_varlen(const void* qkv, const int32_t* cu_seqlens, const void* ctx, const float* lse, const void* keep_mask,
                            const void* dctx, void* dqkv, float* drow, int32_t batch, int32_t max_seq, int32_t total, int32_t heads,
                            int32_t hidden, float dropout_p, uint64_t dropout_seed, uint32_t dropout_stream, void* stream);
/* Attention maps (the tensor output_attention_weights returns, M.py:241-247, 258-259): probs fp32 [batch, heads, seq, seq],
 * probs[b,h,i,j] = softmax_j(q_i . k_j / 8 + mask_bias[b,j]) from the bf16 Q and K of qkv (laid out as for vb_attention_fwd),
 * BEFORE dropout. Every element is written; masked keys (-10000) come out as exact zeros, and an example whose keys are all
 * masked gets softmax(QK^T / 8) over all keys. The kernel computes its own row statistics (it does not read the forward's
 * lse), so the maps are accurate to fp32 rounding for every mask. The argument checks of vb_attention_fwd apply (head_dim 64,
 * qkv 16-byte aligned). */
int vb_attention_probs(const void* qkv, const float* mask_bias, float* probs, int32_t batch, int32_t seq, int32_t heads,
                       int32_t hidden, void* stream);

/* ---- helpers ----------------------------------------------------------------------------- */
/* (1 - cat(input_mask, image_mask)) * -10000 -> fp32 [batch, text+regions]  (M.py:1417, 1286-1294);
 * masks are int64 as the reference dataloaders produce them; image_mask may be NULL (all ones).
 * The casts and the column sum move 16-byte vectors: src and dst of a cast, and x of vb_colsum_bf16, must be 16-byte aligned,
 * and the column sum's ld a multiple of 8 that is >= cols; a call that breaks this returns an error. vb_cast_multi takes any
 * alignment (a misaligned item is cast one element at a time). */
int vb_mask_bias(const int64_t* input_mask, const int64_t* image_mask, float* out, int32_t batch, int32_t text_len,
                 int32_t num_regions, void* stream);
int vb_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream); /* n % 8 == 0 */
int vb_cast_bf16_to_f32(const void* src, float* dst, int64_t n, void* stream);
/* Multi-tensor cast: one launch refreshes every bf16 compute copy (dst_fp32 = 0) and fp32 side copy (dst_fp32 = 1, e.g.
 * the packed q|k|v bias) of a model from its fp32 master parameters. `table` lives in DEVICE memory, ordered by
 * first_chunk; tensor i owns chunks [first_chunk, first_chunk + ceil(numel / VB_CAST_CHUNK)); n_chunks = their total.
 * Replaces the implicit per-step .to(dtype) / fp16 master-copy handling around the reference forward
 * (visualbert/models/train.py:122-136); called at the start of every training-mode forward so that ANY optimizer that
 * changes the masters (the reference BertAdam updates through p.data, optimization.py:293) is seen. */
#define VB_CAST_CHUNK 8192
typedef struct {
    const void* src;   /* fp32 master */
    void* dst;         /* bf16 (or fp32) copy */
    int64_t numel;
    int32_t first_chunk;
    int32_t dst_fp32;
} vb_cast_item;        /* 32 bytes */
int vb_cast_multi(const vb_cast_item* table, int32_t n_items, int32_t n_chunks, void* stream);
int vb_colsum_bf16(const void* x, int64_t ld, float* out, int32_t rows, int32_t cols, void* stream); /* out += */

/* ---- masked-LM loss (M.py:1471-1473, CrossEntropyLoss(ignore_index=-1) on the labelled rows) ------------- */
/* logits bf16 [rows, ld] with valid columns [0, vocab); labels int64 [rows] in [0, vocab).
 * fwd: lse[row] = logsumexp(logits[row, :vocab]), loss_rows[row] = lse - logits[row, label].
 * bwd: logits[row, c] <- (softmax - onehot) * (*scale) for c < vocab and 0 for vocab <= c < padded_cols, IN PLACE
 *      (scale is a device scalar: upstream gradient / number of labelled rows).
 * Labels outside [0, vocab) contribute no loss and no gradient. logits must be 16-byte aligned (ld a multiple of 8); a call
 * with a logits pointer that is not returns an error. rows = 0 launches nothing. */
int vb_cross_entropy_fwd(const void* logits, int64_t ld, const int64_t* labels, int32_t rows, int32_t vocab, float* lse,
                         float* loss_rows, void* stream);
int vb_cross_entropy_bwd(void* logits, int64_t ld, const int64_t* labels, int32_t rows, int32_t vocab, int32_t padded_cols,
                         const float* lse, const float* scale, void* stream);

/* ---- BertLayer (M.py:322-341) ------------------------------------------------------------ */
typedef struct {
    int32_t batch, seq, hidden, heads, inter;
    float hidden_dropout, attn_dropout; /* 0 in eval mode */
    uint64_t seed;                      /* dropout seed of this step */
    uint32_t layer_index;               /* selects the dropout streams of this layer */
    /* bf16 compute copies of the nn.Linear weights ([out, in]) */
    const void* w_qkv;      /* [3H, H]: query | key | value rows (M.py:219-221) */
    const void* w_attn_out; /* [H, H]   attention.output.dense   (M.py:266) */
    const void* w_inter;    /* [I, H]   intermediate.dense       (M.py:298) */
    const void* w_out;      /* [H, I]   output.dense             (M.py:311) */
    /* fp32 vectors */
    const float* b_qkv;     /* [3H] */
    const float* b_attn_out; const float* ln1_gamma; const float* ln1_beta; /* [H] */
    const float* b_inter;   /* [I] */
    const float* b_out; const float* ln2_gamma; const float* ln2_beta;      /* [H] */
    const float* mask_bias; /* [batch, seq] */
} vb_layer_desc;

/* activations written by forward and consumed by backward; M = batch*seq rows, bf16 unless noted */
typedef struct {
    void* qkv;   /* [M, 3H] */
    void* ctx;   /* [M, H]  */
    float* lse;  /* [batch, heads, seq] fp32 */
    void* pre1;  /* [M, H]  attention.output.dense(ctx) (+dropout) + x          (M.py:271-273 before LN) */
    float* mean1; float* rstd1; /* [M] fp32 */
    void* x1;    /* [M, H]  attention output = LN(pre1) */
    void* u;     /* M * I bf16: gelu'(u), u = intermediate.dense(x1) — the derivative is what backward needs. Private to the
                    library (row-major [M, I], or tile-native when vb_gemm_gp_tiled_ok(M, I): see vb_gemm_args.gp_tiled) */
    void* g;     /* [M, I]  gelu(u) */
    void* pre2;  /* [M, H]  output.dense(g) (+dropout) + x1                      (M.py:316-318 before LN) */
    float* mean2; float* rstd2;
    void* keep_mask; /* vb_attention_keep_bytes(batch, seq, heads) bytes; only touched when attn_dropout > 0 */
} vb_layer_acts;

/* fp32 parameter-gradient accumulators (+=), nn.Linear layout. A NULL field is not computed (a frozen parameter): a NULL dw_*
 * skips that weight-gradient GEMM, a NULL db_qkv / db_inter that column sum. A LayerNorm backward forms dgamma, dbeta and the
 * bias gradient of the Linear in front of it in one pass, so (dln1_gamma, dln1_beta, db_attn_out) and (dln2_gamma, dln2_beta,
 * db_out) are each all set or all NULL; all NULL runs that LayerNorm backward without column reductions (and without its
 * deterministic-mode partials), a partly NULL group is refused. Holds for vb_layer_bwd, vb_encoder_bwd and
 * vb_encoder_bwd_varlen in every mode. */
typedef struct {
    float* dw_qkv; float* db_qkv; float* dw_attn_out; float* db_attn_out; float* dln1_gamma; float* dln1_beta;
    float* dw_inter; float* db_inter; float* dw_out; float* db_out; float* dln2_gamma; float* dln2_beta;
} vb_layer_grads;

/* backward scratch, bf16 unless noted */
typedef struct {
    void* d_pre;      /* [M, H] */
    void* d_pre_drop; /* [M, H], only touched when hidden_dropout > 0 */
    void* d_big;      /* [M, max(I, 3H)] */
    void* d_x1;       /* [M, H] */
    void* d_ctx;      /* [M, H] */
    float* drow;      /* [batch, heads, seq] fp32 */
} vb_layer_scratch;

/* x_in, x_out: bf16 [M, H]. x_out = BertLayer(x_in). */
int vb_layer_fwd(const vb_layer_desc* d, const void* x_in, void* x_out, const vb_layer_acts* acts, void* stream);
/* dy: gradient w.r.t. x_out; dx: gradient w.r.t. x_in (may alias dy). dx may be NULL: the input gradient is not needed, and the
 * input-gradient GEMM of the QKV projection (with its residual addend) is not launched. */
int vb_layer_bwd(const vb_layer_desc* d, const void* x_in, const vb_layer_acts* acts, const void* dy, void* dx,
                 const vb_layer_grads* grads, const vb_layer_scratch* scratch, void* stream);

/* ---- BertEncoder (M.py:344-371): the whole layer stack in ONE call -------------------------------------------
 * The per-layer activations (everything vb_layer_acts names, plus each layer's output) live in ONE caller-owned arena
 * whose layout the library defines: vb_encoder_arena_layout fills the byte offsets of the 14 per-layer buffers inside a
 * layer slot (order: qkv, ctx, lse, pre1, mean1, rstd1, x1, u, g, pre2, mean2, rstd2, keep_mask, y) and returns the
 * slot stride; layer l's buffer i sits at arena + l * stride + offsets[i]; total size = n_layers * stride. The same
 * arena pointer is handed to forward and backward (PyTorch owns it; the library allocates nothing). One call replaces
 * the Python loop of M.py:365-368 and its per-layer allocations: host time per step drops to a few calls, and the
 * recurring pointers make the library's tensor-map cache hit.
 * descs[l].seed / dropouts / layer_index are honoured per layer; descs is a HOST array. */
#define VB_ENCODER_ARENA_BUFFERS 14
int64_t vb_encoder_arena_layout(int32_t batch, int32_t seq, int32_t hidden, int32_t heads, int32_t inter, int32_t attn_dropout_on,
                                int64_t* offsets /* [VB_ENCODER_ARENA_BUFFERS] */);
/* x_in bf16 [M, H]; the output of layer l is arena buffer 13 (y) of slot l. */
int vb_encoder_fwd(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* arena, void* stream);
/* dy: gradient w.r.t. the LAST layer's output; dx: gradient w.r.t. x_in; grads: HOST array [n_layers] (NULL fields: see
 * vb_layer_grads; every entry is checked before the first launch). dx may be NULL (also in vb_encoder_bwd_varlen): the lowest
 * layer's input-gradient GEMM is not launched, and the gradient between layers travels in scratch->d_x1 instead of dx. */
int vb_encoder_bwd(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* arena, const void* dy, void* dx,
                   const vb_layer_grads* grads, const vb_layer_scratch* scratch, void* stream);
/* The attention maps of every layer of a dense vb_encoder_fwd call (analysis mode, M.py:1316-1324, 1430-1444): probs fp32
 * [n_layers, batch, heads, seq, seq] = vb_attention_probs of each layer, from the qkv buffer of its arena slot and its
 * descs[l].mask_bias. Call it on the arena and descriptors vb_encoder_fwd just used, before anything overwrites the arena;
 * one launch per layer, no other arena buffer is read. */
int vb_encoder_attention_probs(const vb_layer_desc* descs, int32_t n_layers, void* arena, float* probs, void* stream);
/* Forward-only encoder: the forward of a call that no backward follows — the reference's evaluation loop runs the model under
 * torch.no_grad() (visualbert/models/train.py:292-325). Every layer runs through ONE caller-owned workspace the size of less
 * than one arena slot, whatever n_layers is. Per layer the launches, their arguments and so every output bit are those of
 * vb_encoder_fwd, except that nothing only a backward reads is stored: the FFN-up GEMM uses VB_EPI_GELU_FWD (no gelu'), the
 * attention writes no lse and the LayerNorms no mean / rstd. Dropout (descs[l].hidden_dropout / attn_dropout / seed) is
 * honoured as in vb_encoder_fwd, so the same seed gives the same output.
 * vb_encoder_infer_workspace: bytes of that workspace (a multiple of 256; never more than the arena slot stride of the same
 * shape); packed_rows < 0: dense (M = batch * seq rows), else the row count of a variable-length call with seq = max_seq.
 * Returns -1 on a bad shape.
 * y_last: bf16 [M, hidden], the last layer's output. y_all: NULL, or bf16 [n_layers, M, hidden] receiving every layer's
 * output; y_last must then be NULL or the last slice of y_all. At least one of the two is given.
 * probs: NULL, or fp32 [n_layers, batch, heads, seq, seq] attention maps (dense only; what vb_encoder_attention_probs gives),
 * written per layer from the qkv in the workspace before the next layer overwrites it. */
int64_t vb_encoder_infer_workspace(int32_t batch, int32_t seq, int32_t hidden, int32_t heads, int32_t inter,
                                   int32_t attn_dropout_on, int64_t packed_rows);
int vb_encoder_infer(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* workspace, void* y_last, void* y_all,
                     float* probs, void* stream);
/* Variable-length ("unpadded") encoder: the same calls over `total` packed rows (see vb_attention_fwd_varlen for cu_seqlens and
 * its caller contract). descs[l].batch is the number of sequences and descs[l].seq the longest length (max_seq); mask_bias is
 * ignored and may be NULL. x_in, dy, dx and every row-sized arena / scratch buffer have `total` rows; lse and scratch.drow are
 * fp32 [heads, total]; the keep bits are laid out for (batch, max_seq). The layout returns -1 on a bad shape. total must be
 * > 0 for the forward and backward. */
int64_t vb_encoder_arena_layout_varlen(int32_t batch, int32_t max_seq, int32_t total, int32_t hidden, int32_t heads, int32_t inter,
                                       int32_t attn_dropout_on, int64_t* offsets /* [VB_ENCODER_ARENA_BUFFERS] */);
int vb_encoder_fwd_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total, const void* x_in,
                          void* arena, void* stream);
int vb_encoder_bwd_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total, const void* x_in,
                          void* arena, const void* dy, void* dx, const vb_layer_grads* grads, const vb_layer_scratch* scratch,
                          void* stream);
/* vb_encoder_infer over packed rows: workspace of vb_encoder_infer_workspace with packed_rows = total; y_last bf16 [total, hidden],
 * y_all NULL or bf16 [n_layers, total, hidden]. There are no attention maps of a variable-length call. */
int vb_encoder_infer_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total,
                            const void* x_in, void* workspace, void* y_last, void* y_all, void* stream);
/* Activation checkpointing: a training forward and backward over ONE arena slot (`slot`: vb_encoder_arena_layout bytes, or
 * vb_encoder_arena_layout_varlen bytes for the _varlen calls) plus n_layers - 1 checkpoint regions (`ckpt`), instead of an arena
 * of n_layers slots. Region l holds layer l's output y (bf16 [M, hidden]) and its LayerNorm-2 mean and rstd (fp32 [M]).
 * vb_encoder_ckpt_layout: bytes per region (a multiple of 256); offsets (NULL or [3]) receives the byte offsets of y, mean2,
 * rstd2 (256-byte aligned); packed_rows < 0: dense (M = batch * seq), else the row count of a variable-length call. -1 on a bad
 * shape.
 * vb_encoder_fwd_ckpt: layers 0 .. n-2 run as in vb_encoder_infer, through the slot, and write their output and LN2 statistics
 * into their region; the top layer runs the vb_encoder_fwd forward into the slot, its output in slot buffer 13 (y), reading its
 * input from region n-2. probs: NULL, or the attention maps of vb_encoder_infer (dense only), written per layer from the qkv it
 * just produced.
 * vb_encoder_bwd_ckpt: the backward of vb_encoder_bwd with the same arguments' meaning. The top layer's backward reads the slot;
 * each lower layer is recomputed into the slot up to its FFN-down GEMM (no LN2 forward: its output and statistics are in the
 * region) with the launches and dropout streams of vb_encoder_fwd, then run backward. Every output and gradient bit equals the
 * arena calls' in deterministic mode, and vb_set_dropout_offset applies as there. The slot and ckpt of the forward are handed to
 * the backward unchanged; the backward writes the slot and leaves ckpt as it is. n_layers == 1: ckpt may be NULL and the calls
 * are vb_encoder_fwd / vb_encoder_bwd. Every descriptor and gradient entry is checked before the first launch. */
int64_t vb_encoder_ckpt_layout(int32_t batch, int32_t seq, int32_t hidden, int32_t heads, int32_t inter, int64_t packed_rows,
                               int64_t* offsets /* [3] */);
int vb_encoder_fwd_ckpt(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* ckpt, void* slot, float* probs,
                        void* stream);
int vb_encoder_bwd_ckpt(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* ckpt, void* slot, const void* dy,
                        void* dx, const vb_layer_grads* grads, const vb_layer_scratch* scratch, void* stream);
int vb_encoder_fwd_ckpt_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total,
                               const void* x_in, void* ckpt, void* slot, void* stream);
int vb_encoder_bwd_ckpt_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total,
                               const void* x_in, void* ckpt, void* slot, const void* dy, void* dx, const vb_layer_grads* grads,
                               const vb_layer_scratch* scratch, void* stream);
/* Selective recomputation of the FFN intermediates: the arena calls with every layer's gelu'(u) (buffer 7, u) and g = gelu(u)
 * (buffer 8) moved out of the arena into ONE caller-owned buffer `ffn` that all layers share, instead of 2 * M * inter bf16 per
 * slot. ffn holds gelu'(u) at byte 0, in the order vb_encoder_fwd keeps it (tile-native whenever vb_gemm_gp_tiled_ok(M, inter)),
 * and g at byte ffn_bytes / 2.
 * vb_encoder_arena_layout_ffnrc(_varlen): the arguments, offsets and slot stride of vb_encoder_arena_layout(_varlen), with u and g
 * of size 0 in the slot (offsets[7] == offsets[8] == offsets[9]); *ffn_bytes (if not NULL) receives the size of ffn. -1 on a bad
 * shape.
 * vb_encoder_fwd_ffnrc: the launches and arguments of vb_encoder_fwd, except that each layer's FFN-up GEMM writes gelu'(u) and g
 * into ffn and its FFN-down GEMM reads g from there; on return ffn holds the top layer's.
 * vb_encoder_bwd_ffnrc: vb_encoder_bwd on that arena and the same ffn, as the forward left it. The top layer's backward reads ffn as
 * it is; before the backward of each lower layer l the FFN-up GEMM of its forward (VB_EPI_GELU from slot l's x1, same weights,
 * same tiling) rewrites ffn. That is n_layers - 1 extra GEMMs, and every output and gradient bit equals the arena calls' (in
 * deterministic mode for the gradients). Every descriptor and gradient entry is checked before the first launch.
 * vb_encoder_attention_probs reads only each slot's qkv (offset 0 in both layouts) and mask_bias: on an arena of these calls, give
 * it one layer at a time (n_layers = 1, descs + l, arena + l * stride of vb_encoder_arena_layout_ffnrc). */
int64_t vb_encoder_arena_layout_ffnrc(int32_t batch, int32_t seq, int32_t hidden, int32_t heads, int32_t inter,
                                      int32_t attn_dropout_on, int64_t* offsets /* [VB_ENCODER_ARENA_BUFFERS] */,
                                      int64_t* ffn_bytes);
int64_t vb_encoder_arena_layout_ffnrc_varlen(int32_t batch, int32_t max_seq, int32_t total, int32_t hidden, int32_t heads,
                                             int32_t inter, int32_t attn_dropout_on,
                                             int64_t* offsets /* [VB_ENCODER_ARENA_BUFFERS] */, int64_t* ffn_bytes);
int vb_encoder_fwd_ffnrc(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* arena, void* ffn, void* stream);
int vb_encoder_bwd_ffnrc(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* arena, void* ffn, const void* dy,
                         void* dx, const vb_layer_grads* grads, const vb_layer_scratch* scratch, void* stream);
int vb_encoder_fwd_ffnrc_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total,
                                const void* x_in, void* arena, void* ffn, void* stream);
int vb_encoder_bwd_ffnrc_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total,
                                const void* x_in, void* arena, void* ffn, const void* dy, void* dx, const vb_layer_grads* grads,
                                const vb_layer_scratch* scratch, void* stream);

/* ---- BertEmbeddingsWithVisualEmbedding (M.py:1169-1257) ----------------------------------- */
typedef struct {
    int32_t batch, text_len, num_regions, hidden, visual_dim, vocab, max_pos, n_types;
    float eps, dropout; uint64_t seed;
    const int64_t* input_ids;      /* [batch, text_len] */
    const int64_t* token_type_ids; /* [batch, text_len] */
    const int64_t* visual_type;    /* [batch, num_regions] */
    const void* visual_feats;      /* bf16 [batch*num_regions, visual_dim] */
    const void* w_proj;            /* bf16 [hidden, visual_dim]  projection.weight */
    const float* b_proj;           /* [hidden] */
    const float* word; const float* pos; const float* type; const float* pos_vis; const float* type_vis; /* fp32 tables */
    const float* gamma; const float* beta;
    const void* visual_addend;     /* bf16 [batch*num_regions, hidden] or NULL: extra additive term on the visual rows —
                                      the VCR aligned position embeddings of M.py:1223-1245 (mean of the text position
                                      embeddings a region is aligned to). Its gradient is vb_embed_grads.d_vis. */
} vb_embed_desc;

typedef struct {
    void* vis_proj; /* bf16 [batch*num_regions, hidden] scratch: projection output */
    void* pre;      /* bf16 [M, hidden] pre-LayerNorm sum (saved) */
    float* mean; float* rstd; /* [M] */
} vb_embed_acts;

/* A NULL table (dword, dpos, dtype, dpos_vis, dtype_vis) receives no scatter: a frozen table. In deterministic mode its rows
 * still take part in the key sort, so the sum order of every other table is that of the call with every table given, bit for
 * bit. A NULL dw_proj / db_proj skips the projection's weight-gradient GEMM / column sum; dgamma and dbeta both NULL run the
 * embedding LayerNorm backward without column reductions (one of them NULL: that one is not written). */
typedef struct {
    float* dword; float* dpos; float* dtype; float* dpos_vis; float* dtype_vis; /* fp32 tables, += */
    float* dw_proj; float* db_proj; float* dgamma; float* dbeta;
    void* d_pre;  /* bf16 [M, hidden] scratch */
    void* d_vis;  /* bf16 [batch*num_regions, hidden] scratch */
    void* d_feats; /* bf16 [batch*num_regions, visual_dim] or NULL: gradient w.r.t. the region features */
} vb_embed_grads;

/* y: bf16 [M, hidden] = dropout(LN(cat(text, visual))). Ids and types outside their tables are clamped to the first or last
 * row. The fp32 tables are read as 16-byte vectors: word, pos, type, pos_vis, type_vis, and acts->pre, acts->vis_proj and y, must
 * be 16-byte aligned; in the backward dword, dpos and d_vis must be. A call that breaks this returns an error before launching. */
int vb_embed_fwd(const vb_embed_desc* d, void* y, const vb_embed_acts* acts, void* stream);
int vb_embed_bwd(const vb_embed_desc* d, const vb_embed_acts* acts, const void* dy, const vb_embed_grads* g, void* stream);

/* ---- BertAdam (SURVEY.md §8f rank 2) ------------------------------------------------------------------------
 * Replaces the per-tensor Python loop of BertAdam.step, visualbert/pytorch_pretrained_bert/optimization.py:239-304:
 * Adam WITHOUT bias correction (opt.py:299-302), decoupled weight decay added to the update (opt.py:287-288),
 * gradient clipping PER PARAMETER TENSOR to max_grad_norm (opt.py:272-273, torch clip_grad_norm_ semantics:
 * coef = max_norm / (||g||_2 + 1e-6), applied when < 1), learning rate already multiplied by the schedule value of
 * the tensor's own step counter (opt.py:290-291) by the caller. One call = one optimizer step over all tensors of a
 * table that lives in DEVICE memory; two launches (per-tensor sum of squares, update). Gradients are read, never
 * modified (the reference scales p.grad in place as a side effect of the clip; callers zero it afterwards). */
#define VB_ADAM_CHUNK 32768 /* elements per CTA; tensor i owns chunks [first_chunk, first_chunk + ceil(numel/CHUNK)) */
typedef struct {
    void* p;          /* fp32 parameter, updated in place */
    const void* g;    /* fp32 gradient */
    void* m;          /* fp32 next_m (state['next_m'], opt.py:262) */
    void* v;          /* fp32 next_v (state['next_v'], opt.py:264) */
    int64_t numel;
    float lr;           /* group lr * schedule.get_lr(state['step']) */
    float weight_decay; /* group weight_decay (0 for the bias / LayerNorm group, model_wrapper.py:106-111) */
    int32_t first_chunk;
    int32_t reserved;   /* vb_bert_adam_step: ignored. vb_bert_adam_step_sched: the tensor's group, an index into `groups` */
} vb_adam_tensor;     /* 56 bytes */
/* table: device array [n_tensors] ordered by first_chunk; sumsq: device scratch [n_tensors] (overwritten).
 * b1/b2/eps/max_grad_norm are doubles because the reference forms (1 - b) in double precision; max_grad_norm <= 0
 * disables clipping (opt.py:272). */
int vb_bert_adam_step(const vb_adam_tensor* table, int32_t n_tensors, int32_t n_chunks, float* sumsq, double b1, double b2,
                      double eps, double max_grad_norm, void* stream);

/* BertAdam with the learning-rate schedule evaluated on the device (CUDA graphs). The same step as vb_bert_adam_step, with the
 * same bits, except that each tensor's lr and weight decay come from its group and its own step counter when the kernels run:
 *   lr = fp32(groups[g].lr * schedule(steps[t] / t_total))  (fp64, the operation order of optimization.py, one rounding to fp32)
 * with g = table[t].reserved; table[t].lr and table[t].weight_decay are ignored. Every CTA of a tensor uses the step value from
 * before the call, and the call then advances each of the n_tensors counters by exactly one (a third, small launch). Nothing is
 * read back on the host, so a captured call replayed later reads the counters and the group table as they are then. */
#define VB_SCHED_CONSTANT 0        /* ConstantLR: 1 */
#define VB_SCHED_WARMUP_CONSTANT 1 /* WarmupConstantSchedule: x / warmup while x < warmup, then 1 */
#define VB_SCHED_WARMUP_LINEAR 2   /* WarmupLinearSchedule: x / warmup, then max((x - 1) / (warmup - 1), 0) */
#define VB_SCHED_WARMUP_COSINE 3   /* WarmupCosineSchedule: x / warmup, then 0.5 (1 + cos(pi cycles 2 (x - warmup) / (1 - warmup))) */
typedef struct {
    double lr;          /* the group's base lr (group['lr']) */
    double warmup;      /* fraction of t_total, already max(warmup, 0), < 1 */
    double t_total;     /* < 0: the multiplier is 1 whatever the kind; 0 is refused (the host schedule divides by it) */
    double cycles;      /* VB_SCHED_WARMUP_COSINE only */
    float weight_decay; /* fp32, as vb_adam_tensor.weight_decay */
    int32_t schedule;   /* VB_SCHED_* */
} vb_adam_group;        /* 40 bytes */
/* table, groups: device arrays [n_tensors] (as for vb_bert_adam_step) and [n_groups]; steps: device int64 [n_tensors], the step
 * counter of each tensor (state['step']), read and then advanced by one; sumsq: device scratch [n_tensors]; lr_out: NULL, or a
 * device float [n_tensors] that receives the lr each tensor was updated with. In deterministic mode (vb_set_deterministic) the
 * gradient norms take the fixed-order path, as in vb_bert_adam_step. The call checks its pointers, counts and b1 / b2 / eps; the
 * contents of the device tables cannot be read on the host without a copy that a graph would freeze, so they are checked by
 * vb_bert_adam_sched_check on the host copies the caller uploads. */
int vb_bert_adam_step_sched(const vb_adam_tensor* table, int32_t n_tensors, int32_t n_chunks, const vb_adam_group* groups,
                            int32_t n_groups, int64_t* steps, float* sumsq, float* lr_out, double b1, double b2, double eps,
                            double max_grad_norm, void* stream);
/* Host-side check of the tables vb_bert_adam_step_sched will read, on the HOST copies before they are uploaded: the chunk layout
 * (first_chunk in order, n_chunks covering every tensor), each tensor's group index in [0, n_groups), each group's schedule kind,
 * warmup in [0, 1) and t_total != 0. No CUDA call. */
int vb_bert_adam_sched_check(const vb_adam_tensor* table, int32_t n_tensors, int32_t n_chunks, const vb_adam_group* groups,
                             int32_t n_groups);

#ifdef __cplusplus
}
#endif
#endif /* VBERT_B200_H */
