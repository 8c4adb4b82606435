// vb_api.cu — layer-level entry points of the C ABI: one call launches every kernel of a BertLayer
// forward (8 launches with attention dropout) or backward (13 launches), or of the visual+text embedding block.
//
// Kernel sequence of vb_layer_fwd (reference modeling.py:331-341):
//   1 GEMM   qkv  = x Wqkv^T + b                       (M.py:232-234, three Linears fused into N = 3H)
//   2 ATTN   ctx  = softmax(QK^T/8 + mask) V           (M.py:241-256)
//   3 GEMM   pre1 = dropout(ctx Wo^T + b) + x          (M.py:271-273, bias/dropout/residual in the epilogue)
//   4 LN     x1   = LayerNorm(pre1)                    (M.py:273)
//   5 GEMM   u, g = x1 W1^T + b, gelu(u)               (M.py:303-304, GELU in the epilogue)
//   6 GEMM   pre2 = dropout(g W2^T + b) + x1           (M.py:316-318)
//   7 LN     out  = LayerNorm(pre2)
// vb_layer_bwd is the exact adjoint (autograd of the above), weight gradients accumulated in fp32.
// vb_encoder_infer runs the same sequence for a forward no backward follows: step 5 writes g alone and no statistics are kept.
#include <string.h>

#include "vb_internal.h"

namespace vb {

constexpr float kLnEps = 1e-12f;
constexpr unsigned kEmbedDropStream = 0xE0000001u;
enum { kSiteAttnProbs = 0, kSiteAttnOut = 1, kSiteFfnOut = 2 };
static inline unsigned drop_stream(unsigned layer, unsigned site) { return layer * 8u + site; }

#define VB_TRY(expr)            \
    do {                        \
        int _rc = (expr);       \
        if (_rc) return _rc;    \
    } while (0)

// y[M,N] (bf16) = epi(A[M,K] W[N,K]^T)
static vb_gemm_args fwd_args(const void* A, const void* W, void* D, int M, int N, int K) {
    vb_gemm_args a;
    memset(&a, 0, sizeof(a));
    a.A = A; a.lda = K; a.B = W; a.ldb = K; a.M = M; a.N = N; a.K = K; a.D = D; a.ldd = N;
    return a;
}
// dX[M,K] (bf16) = dY[M,N] W[N,K]
static vb_gemm_args dgrad_args(const void* dY, const void* W, void* dX, int M, int N, int K) {
    vb_gemm_args a;
    memset(&a, 0, sizeof(a));
    a.A = dY; a.lda = N; a.B = W; a.ldb = K; a.b_mn_major = 1; a.M = M; a.N = K; a.K = N; a.D = dX; a.ldd = K;
    return a;
}
// dW[N,K] (fp32, +=) = dY[M,N]^T X[M,K]
static vb_gemm_args wgrad_args(const void* dY, const void* X, float* dW, int M, int N, int K) {
    vb_gemm_args a;
    memset(&a, 0, sizeof(a));
    a.A = dY; a.lda = N; a.a_mn_major = 1; a.B = X; a.ldb = K; a.b_mn_major = 1;
    a.M = N; a.N = K; a.K = M; a.D = dW; a.ldd = K; a.d_fp32 = 1;
    return a;
}

// The rows a layer call works on. Dense: batch * seq rows, sequence b at rows b * seq. Variable-length ("unpadded"): `total`
// packed rows, sequence b at rows [cu_seqlens[b], cu_seqlens[b + 1]) (device memory), at most seq (the longest) rows each;
// the attention runs through the varlen kernels, everything else is row-local and only sees M = total.
struct LayerRows {
    const int* cu_seqlens;  // nullptr: dense
    int total;
};
static const LayerRows kDenseRows = {nullptr, 0};

static int check_layer(const vb_layer_desc* d, const LayerRows& r) {
    VB_REQUIRE(d != nullptr, "layer: null descriptor");
    VB_REQUIRE(d->batch > 0 && d->seq > 0, "layer: empty batch");
    VB_REQUIRE(d->hidden == d->heads * 64, "layer: hidden (%d) must equal heads (%d) * 64", d->hidden, d->heads);
    VB_REQUIRE(d->hidden % 16 == 0 && d->inter % 16 == 0, "layer: hidden/intermediate must be multiples of 16");
    VB_REQUIRE(d->w_qkv && d->w_attn_out && d->w_inter && d->w_out, "layer: null weight pointer");
    VB_REQUIRE(r.cu_seqlens != nullptr || d->mask_bias != nullptr, "layer: null mask_bias");
    VB_REQUIRE(r.cu_seqlens == nullptr || r.total > 0, "layer: varlen call without rows (total = %d)", r.total);
    return 0;
}

// for_bwd = false (vb_encoder_infer): the same launches with the same arguments, but nothing only a backward reads is stored —
// s->u is not touched (the FFN-up epilogue writes gelu(u) alone) and s->lse, s->mean1/2, s->rstd1/2 may be NULL
int layer_fwd(const vb_layer_desc* d, const void* x_in, void* x_out, const vb_layer_acts* s, cudaStream_t st,
              const LayerRows& rows = kDenseRows, bool for_bwd = true) {
    VB_TRY(check_layer(d, rows));
    VB_REQUIRE(x_in && x_out && s, "layer_fwd: null pointer");
    const bool vl = rows.cu_seqlens != nullptr;
    const int M = vl ? rows.total : d->batch * d->seq, H = d->hidden, I = d->inter;
    vb_gemm_args a = fwd_args(x_in, d->w_qkv, s->qkv, M, 3 * H, H);
    a.bias = d->b_qkv;
    VB_TRY(gemm(a, st));
    if (vl)
        VB_TRY(attn_fwd_varlen(s->qkv, rows.cu_seqlens, s->ctx, s->lse, s->keep_mask, d->batch, d->seq, rows.total, d->heads, H,
                               d->attn_dropout, d->seed, drop_stream(d->layer_index, kSiteAttnProbs), st, for_bwd));
    else
        VB_TRY(attn_fwd(s->qkv, d->mask_bias, s->ctx, s->lse, s->keep_mask, d->batch, d->seq, d->heads, H, d->attn_dropout, d->seed,
                        drop_stream(d->layer_index, kSiteAttnProbs), st));
    a = fwd_args(s->ctx, d->w_attn_out, s->pre1, M, H, H);
    a.bias = d->b_attn_out; a.addend = x_in; a.ld_add = H;
    a.dropout_p = d->hidden_dropout; a.dropout_seed = d->seed; a.dropout_stream = drop_stream(d->layer_index, kSiteAttnOut);
    VB_TRY(gemm(a, st));
    VB_TRY(ln_fwd(s->pre1, H, d->ln1_gamma, d->ln1_beta, s->x1, H, s->mean1, s->rstd1, M, H, kLnEps, st));
    if (for_bwd) {
        a = fwd_args(s->x1, d->w_inter, s->u, M, I, H);
        a.bias = d->b_inter; a.epilogue = VB_EPI_GELU; a.aux_out = s->g; a.ld_aux = I;
        a.gp_tiled = gemm_gp_tiled_ok(M, I) ? 1 : 0;   // acts.u is private to the library: tile-native whenever the shape allows
    } else {
        a = fwd_args(s->x1, d->w_inter, s->g, M, I, H);
        a.bias = d->b_inter; a.epilogue = VB_EPI_GELU_FWD;
    }
    VB_TRY(gemm(a, st));
    a = fwd_args(s->g, d->w_out, s->pre2, M, H, I);
    a.bias = d->b_out; a.addend = s->x1; a.ld_add = H;
    a.dropout_p = d->hidden_dropout; a.dropout_seed = d->seed; a.dropout_stream = drop_stream(d->layer_index, kSiteFfnOut);
    VB_TRY(gemm(a, st));
    VB_TRY(ln_fwd(s->pre2, H, d->ln2_gamma, d->ln2_beta, x_out, H, s->mean2, s->rstd2, M, H, kLnEps, st));
    return 0;
}

// deterministic mode: the workspace one layer backward needs (its LayerNorm and column-sum partials; a weight-gradient GEMM
// whose slabs do not fit lowers its split factor instead). Checked before the first launch, so a refused call launches nothing.
static long long layer_bwd_det_bytes(int M, int H, int I) {
    const long long c = colsum_det_bytes(M, I) > colsum_det_bytes(M, 3 * H) ? colsum_det_bytes(M, I) : colsum_det_bytes(M, 3 * H);
    return ln_bwd_det_bytes(M, H) > c ? ln_bwd_det_bytes(M, H) : c;
}

int layer_bwd(const vb_layer_desc* d, const void* x_in, const vb_layer_acts* s, const void* dy, void* dx,
              const vb_layer_grads* g, const vb_layer_scratch* w, cudaStream_t st, const LayerRows& rows = kDenseRows) {
    VB_TRY(check_layer(d, rows));
    VB_REQUIRE(x_in && s && dy && dx && g && w, "layer_bwd: null pointer");
    const bool vl = rows.cu_seqlens != nullptr;
    const int M = vl ? rows.total : d->batch * d->seq, H = d->hidden, I = d->inter;
    VB_TRY(det_require(layer_bwd_det_bytes(M, H, I), "layer backward"));
    const bool hd = d->hidden_dropout > 0.f;
    VB_REQUIRE(!hd || w->d_pre_drop, "layer_bwd: d_pre_drop scratch required when hidden_dropout > 0");
    void* dpm = hd ? w->d_pre_drop : w->d_pre;  // gradient entering the Linear in front of each LayerNorm

    // ---- BertOutput: LN2, output.dense ----
    VB_TRY(ln_bwd(dy, s->pre2, s->mean2, s->rstd2, d->ln2_gamma, w->d_pre, hd ? w->d_pre_drop : nullptr, g->dln2_gamma,
                  g->dln2_beta, g->db_out, M, H, d->hidden_dropout, d->seed, drop_stream(d->layer_index, kSiteFfnOut),
                  0.f, 0, st));
    VB_TRY(gemm(wgrad_args(dpm, s->g, g->dw_out, M, H, I), st));
    vb_gemm_args a = dgrad_args(dpm, d->w_out, w->d_big, M, H, I);  // d_g, then * gelu'(u) -> d_u
    a.epilogue = VB_EPI_DGELU; a.aux_in = s->u; a.ld_aux = I;
    a.gp_tiled = gemm_gp_tiled_ok(M, I) ? 1 : 0;
    VB_TRY(gemm(a, st));
    // ---- BertIntermediate ----
    VB_TRY(colsum(w->d_big, I, g->db_inter, M, I, st));
    VB_TRY(gemm(wgrad_args(w->d_big, s->x1, g->dw_inter, M, I, H), st));
    a = dgrad_args(w->d_big, d->w_inter, w->d_x1, M, I, H);
    a.addend = w->d_pre; a.ld_add = H;  // + residual branch of BertOutput
    VB_TRY(gemm(a, st));
    // ---- BertSelfOutput: LN1, attention.output.dense ----
    VB_TRY(ln_bwd(w->d_x1, s->pre1, s->mean1, s->rstd1, d->ln1_gamma, w->d_pre, hd ? w->d_pre_drop : nullptr,
                  g->dln1_gamma, g->dln1_beta, g->db_attn_out, M, H, d->hidden_dropout, d->seed,
                  drop_stream(d->layer_index, kSiteAttnOut), 0.f, 0, st));
    VB_TRY(gemm(wgrad_args(dpm, s->ctx, g->dw_attn_out, M, H, H), st));
    a = dgrad_args(dpm, d->w_attn_out, w->d_ctx, M, H, H);
    // D = rowsum(dO * O) of the attention backward falls out of this GEMM's epilogue (a thread holds two whole heads of a row);
    // the staged attention kernels compute D themselves
    const bool fused_delta = gemm_delta_ok(M, H) && w->drow != nullptr && attn_route(d->seq) != AttnRoute::Staged;
    // (varlen: drow is [heads, total], i.e. delta_out[0][h][row] with delta_seq = total)
    if (fused_delta) { a.delta_ctx = s->ctx; a.delta_out = w->drow; a.delta_seq = vl ? rows.total : d->seq; }
    VB_TRY(gemm(a, st));
    // ---- BertSelfAttention ----
    if (vl)
        VB_TRY(attn_bwd_varlen(s->qkv, rows.cu_seqlens, s->ctx, s->lse, s->keep_mask, w->d_ctx, w->d_big, w->drow, d->batch, d->seq,
                               rows.total, d->heads, H, d->attn_dropout, d->seed, drop_stream(d->layer_index, kSiteAttnProbs), st,
                               fused_delta));
    else
        VB_TRY(attn_bwd(s->qkv, d->mask_bias, s->ctx, s->lse, s->keep_mask, w->d_ctx, w->d_big, w->drow, d->batch, d->seq, d->heads, H,
                        d->attn_dropout, d->seed, drop_stream(d->layer_index, kSiteAttnProbs), st, fused_delta));
    VB_TRY(colsum(w->d_big, 3 * H, g->db_qkv, M, 3 * H, st));
    VB_TRY(gemm(wgrad_args(w->d_big, x_in, g->dw_qkv, M, 3 * H, H), st));
    a = dgrad_args(w->d_big, d->w_qkv, dx, M, 3 * H, H);
    a.addend = w->d_pre; a.ld_add = H;  // + residual branch of BertSelfOutput
    VB_TRY(gemm(a, st));
    return 0;
}

// ---- whole-encoder entry points: one arena, one call (see include/vbert_b200.h) ----
static long long align256(long long x) { return (x + 255) / 256 * 256; }

// M rows per layer (B * S dense, total varlen); lse holds A * M floats either way ([B, A, S] or [A, total]); the keep bits are
// laid out for (B, S) with S the longest sequence
long long encoder_arena_layout(int B, int S, int H, int A, int I, int attn_drop, long long* off, long long packed_rows = -1) {
    const long long M = packed_rows >= 0 ? packed_rows : static_cast<long long>(B) * S;
    const long long sizes[VB_ENCODER_ARENA_BUFFERS] = {
        M * 3 * H * 2, M * H * 2, static_cast<long long>(A) * M * 4, M * H * 2, M * 4, M * 4, M * H * 2, M * I * 2, M * I * 2,
        M * H * 2, M * 4, M * 4, attn_drop ? attn_keep_bytes(B, S, A) : 0, M * H * 2};
    long long o = 0;
    for (int i = 0; i < VB_ENCODER_ARENA_BUFFERS; ++i) {
        if (off) off[i] = o;
        o += align256(sizes[i]);
    }
    return o;
}

static void arena_acts(const vb_layer_desc* d, void* arena, int l, vb_layer_acts* a, void** y, const LayerRows& rows) {
    long long off[VB_ENCODER_ARENA_BUFFERS];
    const long long stride = encoder_arena_layout(d->batch, d->seq, d->hidden, d->heads, d->inter, d->attn_dropout > 0.f, off,
                                                  rows.cu_seqlens != nullptr ? rows.total : -1);
    char* base = static_cast<char*>(arena) + l * stride;
    a->qkv = base + off[0]; a->ctx = base + off[1]; a->lse = reinterpret_cast<float*>(base + off[2]);
    a->pre1 = base + off[3]; a->mean1 = reinterpret_cast<float*>(base + off[4]); a->rstd1 = reinterpret_cast<float*>(base + off[5]);
    a->x1 = base + off[6]; a->u = base + off[7]; a->g = base + off[8]; a->pre2 = base + off[9];
    a->mean2 = reinterpret_cast<float*>(base + off[10]); a->rstd2 = reinterpret_cast<float*>(base + off[11]);
    a->keep_mask = d->attn_dropout > 0.f ? base + off[12] : nullptr;
    *y = base + off[13];
}

int encoder_fwd(const vb_layer_desc* descs, int n, const void* x_in, void* arena, cudaStream_t st, const LayerRows& rows = kDenseRows) {
    VB_REQUIRE(descs && n > 0 && x_in && arena, "encoder_fwd: null pointer / no layers");
    const void* x = x_in;
    for (int l = 0; l < n; ++l) {
        VB_REQUIRE(descs[l].batch == descs[0].batch && descs[l].seq == descs[0].seq && descs[l].hidden == descs[0].hidden &&
                   descs[l].heads == descs[0].heads && descs[l].inter == descs[0].inter &&
                   (descs[l].attn_dropout > 0.f) == (descs[0].attn_dropout > 0.f), "encoder_fwd: layers differ in shape");
        vb_layer_acts a;
        void* y;
        arena_acts(&descs[l], arena, l, &a, &y, rows);
        VB_TRY(layer_fwd(&descs[l], x, y, &a, st, rows));
        x = y;
    }
    return 0;
}

int encoder_bwd(const vb_layer_desc* descs, int n, const void* x_in, void* arena, const void* dy, void* dx,
                const vb_layer_grads* grads, const vb_layer_scratch* w, cudaStream_t st, const LayerRows& rows = kDenseRows) {
    VB_REQUIRE(descs && n > 0 && x_in && arena && dy && dx && grads && w, "encoder_bwd: null pointer / no layers");
    const void* g_in = dy;
    for (int l = n - 1; l >= 0; --l) {
        vb_layer_acts a;
        void* y;
        arena_acts(&descs[l], arena, l, &a, &y, rows);
        const void* xl = x_in;
        if (l > 0) {
            vb_layer_acts ap;
            void* yp;
            arena_acts(&descs[l - 1], arena, l - 1, &ap, &yp, rows);
            xl = yp;
        }
        // the gradient buffer ping-pongs inside `dx` (vb_layer_bwd allows dx to alias dy)
        VB_TRY(layer_bwd(&descs[l], xl, &a, g_in, dx, &grads[l], w, st, rows));
        g_in = dx;
    }
    return 0;
}

// ---- forward-only encoder: every layer through one workspace, nothing kept for a backward ----
enum { kWsQkv, kWsCtx, kWsPre, kWsX1, kWsG, kWsKeep, kWsY0, kWsY1, kWsBuffers };

// pre1 and pre2 share one buffer (LayerNorm 1 has consumed pre1 before the FFN-down GEMM writes pre2); y0 / y1 are the ping-pong
// layer outputs of a call without y_all. Everything here is also in an arena slot, which holds u, lse and the statistics besides:
// the workspace is never larger than the slot.
long long infer_workspace_layout(int B, int S, int H, int A, int I, int attn_drop, long long packed_rows, long long* off) {
    const long long M = packed_rows >= 0 ? packed_rows : static_cast<long long>(B) * S;
    const long long sizes[kWsBuffers] = {M * 3 * H * 2, M * H * 2, M * H * 2, M * H * 2, M * I * 2,
                                         attn_drop ? attn_keep_bytes(B, S, A) : 0, M * H * 2, M * H * 2};
    long long o = 0;
    for (int i = 0; i < kWsBuffers; ++i) {
        if (off) off[i] = o;
        o += align256(sizes[i]);
    }
    return o;
}

int encoder_infer(const vb_layer_desc* descs, int n, const void* x_in, void* workspace, void* y_last, void* y_all, float* probs,
                  cudaStream_t st, const LayerRows& rows = kDenseRows) {
    VB_REQUIRE(descs && n > 0, "encoder_infer: null descriptors / no layers");
    VB_REQUIRE(x_in && workspace, "encoder_infer: null x_in / workspace");
    VB_REQUIRE(y_last || y_all, "encoder_infer: y_last and y_all are both NULL");
    const vb_layer_desc& d0 = descs[0];
    for (int l = 0; l < n; ++l) {  // every descriptor is checked before the first launch: a refused call writes nothing
        VB_TRY(check_layer(&descs[l], rows));
        VB_REQUIRE(descs[l].batch == d0.batch && descs[l].seq == d0.seq && descs[l].hidden == d0.hidden && descs[l].heads == d0.heads &&
                   descs[l].inter == d0.inter && (descs[l].attn_dropout > 0.f) == (d0.attn_dropout > 0.f),
                   "encoder_infer: layers differ in shape");
    }
    const bool vl = rows.cu_seqlens != nullptr;
    const long long M = vl ? rows.total : static_cast<long long>(d0.batch) * d0.seq;
    const long long y_bytes = M * d0.hidden * 2;
    char* const ya = static_cast<char*>(y_all);
    VB_REQUIRE(!ya || !y_last || y_last == ya + (n - 1) * y_bytes, "encoder_infer: with y_all, y_last must be NULL or its last slice");
    long long off[kWsBuffers];
    infer_workspace_layout(d0.batch, d0.seq, d0.hidden, d0.heads, d0.inter, d0.attn_dropout > 0.f, vl ? rows.total : -1, off);
    char* const ws = static_cast<char*>(workspace);
    vb_layer_acts a;
    memset(&a, 0, sizeof(a));
    a.qkv = ws + off[kWsQkv]; a.ctx = ws + off[kWsCtx]; a.pre1 = a.pre2 = ws + off[kWsPre]; a.x1 = ws + off[kWsX1]; a.g = ws + off[kWsG];
    a.keep_mask = d0.attn_dropout > 0.f ? ws + off[kWsKeep] : nullptr;
    const long long per_layer = static_cast<long long>(d0.batch) * d0.heads * d0.seq * d0.seq;
    const void* x = x_in;
    for (int l = 0; l < n; ++l) {
        void* y = ya ? ya + l * y_bytes : l == n - 1 ? y_last : ws + off[(l & 1) ? kWsY1 : kWsY0];
        VB_TRY(layer_fwd(&descs[l], x, y, &a, st, rows, false));
        if (probs)
            VB_TRY(attn_probs(a.qkv, descs[l].mask_bias, probs + l * per_layer, d0.batch, d0.seq, d0.heads, d0.hidden, st));
        x = y;
    }
    return 0;
}

// the attention maps of every layer of a dense vb_encoder_fwd, from the qkv each layer slot of the arena holds
int encoder_attention_probs(const vb_layer_desc* descs, int n, void* arena, float* probs, cudaStream_t st) {
    VB_REQUIRE(descs && n > 0 && arena && probs, "encoder_attention_probs: null pointer / no layers");
    for (int l = 0; l < n; ++l) {  // every descriptor is checked before the first launch: a refused call writes nothing
        VB_TRY(check_layer(&descs[l], kDenseRows));
        VB_REQUIRE(descs[l].batch == descs[0].batch && descs[l].seq == descs[0].seq && descs[l].hidden == descs[0].hidden &&
                   descs[l].heads == descs[0].heads && descs[l].inter == descs[0].inter &&
                   (descs[l].attn_dropout > 0.f) == (descs[0].attn_dropout > 0.f), "encoder_attention_probs: layers differ in shape");
    }
    const long long per_layer = static_cast<long long>(descs[0].batch) * descs[0].heads * descs[0].seq * descs[0].seq;
    for (int l = 0; l < n; ++l) {
        vb_layer_acts a;
        void* y;
        arena_acts(&descs[l], arena, l, &a, &y, kDenseRows);
        VB_TRY(attn_probs(a.qkv, descs[l].mask_bias, probs + l * per_layer, descs[l].batch, descs[l].seq, descs[l].heads,
                          descs[l].hidden, st));
    }
    return 0;
}

static int check_embed(const vb_embed_desc* d) {
    VB_REQUIRE(d != nullptr, "embed: null descriptor");
    VB_REQUIRE(d->batch > 0 && d->text_len > 0 && d->num_regions >= 0, "embed: bad shape");
    VB_REQUIRE(d->hidden % 16 == 0, "embed: hidden must be a multiple of 16");
    VB_REQUIRE(d->num_regions == 0 || (d->visual_dim % 8 == 0 && d->visual_feats && d->w_proj && d->visual_type),
               "embed: visual inputs missing or visual_dim not a multiple of 8");
    return 0;
}

int embed_fwd_api(const vb_embed_desc* d, void* y, const vb_embed_acts* s, cudaStream_t st) {
    VB_TRY(check_embed(d));
    VB_REQUIRE(y && s && s->pre && s->mean && s->rstd, "embed_fwd: null pointer");
    const int BV = d->batch * d->num_regions;
    if (BV > 0) {
        vb_gemm_args a = fwd_args(d->visual_feats, d->w_proj, s->vis_proj, BV, d->hidden, d->visual_dim);
        a.bias = d->b_proj;
        if (d->visual_addend != nullptr) {  // aligned position embeddings ride the projection GEMM's residual input
            a.addend = d->visual_addend;
            a.ld_add = d->hidden;
        }
        VB_TRY(gemm(a, st));
    }
    EmbedParams p;
    memset(&p, 0, sizeof(p));
    p.ids = reinterpret_cast<const long long*>(d->input_ids);
    p.tt = reinterpret_cast<const long long*>(d->token_type_ids);
    p.vt = reinterpret_cast<const long long*>(d->visual_type);
    p.vis_proj = static_cast<const bf16*>(s->vis_proj);
    p.word = d->word; p.pos = d->pos; p.type = d->type; p.pos_vis = d->pos_vis; p.type_vis = d->type_vis;
    p.gamma = d->gamma; p.beta = d->beta;
    p.pre = static_cast<bf16*>(s->pre); p.y = static_cast<bf16*>(y); p.mean = s->mean; p.rstd = s->rstd;
    p.B = d->batch; p.T = d->text_len; p.V = d->num_regions; p.H = d->hidden;
    p.vocab = d->vocab; p.max_pos = d->max_pos; p.n_types = d->n_types;
    p.eps = d->eps;
    if (d->dropout > 0.f) {
        const DropQ q = dropout_quantise(d->dropout);
        p.drop_scale = q.scale;
        p.drop_thresh16 = q.thr8;
        p.drop_seed = d->seed;
        p.drop_stream = kEmbedDropStream;
    }
    return embed_fwd(p, st);
}

int embed_bwd_api(const vb_embed_desc* d, const vb_embed_acts* s, const void* dy, const vb_embed_grads* g,
                  cudaStream_t st) {
    VB_TRY(check_embed(d));
    VB_REQUIRE(s && dy && g && g->d_pre, "embed_bwd: null pointer");
    const int M = d->batch * (d->text_len + d->num_regions), H = d->hidden, BV = d->batch * d->num_regions;
    if (det_ws().ptr != nullptr) {   // every launch of the call fits the workspace, or nothing is launched
        const long long temp = embed_sort_temp_bytes(d->batch, d->text_len, d->num_regions);
        VB_REQUIRE(temp >= 0, "embed_bwd: radix sort size query failed");
        long long need = embed_bwd_det_bytes(d->batch, d->text_len, d->num_regions, H, temp);
        if (ln_bwd_det_bytes(M, H) > need) need = ln_bwd_det_bytes(M, H);
        if (BV > 0 && colsum_det_bytes(BV, H) > need) need = colsum_det_bytes(BV, H);
        VB_TRY(det_require(need, "embed_bwd"));
    }
    VB_TRY(ln_bwd(dy, s->pre, s->mean, s->rstd, d->gamma, g->d_pre, nullptr, g->dgamma, g->dbeta, nullptr, M, H, 0.f,
                  d->seed, 0, d->dropout, kEmbedDropStream, st));
    EmbedBwdParams p;
    memset(&p, 0, sizeof(p));
    p.de = static_cast<const bf16*>(g->d_pre);
    p.ids = reinterpret_cast<const long long*>(d->input_ids);
    p.tt = reinterpret_cast<const long long*>(d->token_type_ids);
    p.vt = reinterpret_cast<const long long*>(d->visual_type);
    p.dword = g->dword; p.dpos = g->dpos; p.dtype = g->dtype; p.dpos_vis = g->dpos_vis; p.dtype_vis = g->dtype_vis;
    p.dvis = static_cast<bf16*>(g->d_vis);
    p.B = d->batch; p.T = d->text_len; p.V = d->num_regions; p.H = H;
    p.vocab = d->vocab; p.max_pos = d->max_pos; p.n_types = d->n_types;
    VB_TRY(embed_bwd(p, st));
    if (BV > 0) {
        VB_TRY(colsum(g->d_vis, H, g->db_proj, BV, H, st));
        VB_TRY(gemm(wgrad_args(g->d_vis, d->visual_feats, g->dw_proj, BV, H, d->visual_dim), st));
        if (g->d_feats) VB_TRY(gemm(dgrad_args(g->d_vis, d->w_proj, g->d_feats, BV, H, d->visual_dim), st));
    }
    return 0;
}

// vb_deterministic_workspace_bytes: the largest workspace any deterministic call of these shapes takes, as a function that grows
// with every argument. A weight-gradient GEMM's slabs are sized for the split factor of every K up to `rows` (so that none of these
// GEMMs lowers its split factor, and the bits do not depend on which calls sized the workspace first); the split factor falls as
// the tile count grows, so the MLM decoder's [vocab, H] term is the largest over every smaller padded vocabulary. Column sums are
// bounded by 4 * max(N, 6 * SMs * 256) bytes (colsum_gy partial rows of N columns).
static int max_splits(long long tiles, int rows) {
    int splits = 1;
    for (int kb = 1; kb <= gemm_k_blocks(rows); ++kb) { const int s = wgrad_splits(tiles, kb); if (s > splits) splits = s; }
    return splits;
}
long long deterministic_workspace_bytes(long long rows, int H, int I, int vocab, int adam_chunks) {
    long long need = 4LL * adam_chunks;
    auto up = [&](long long b) { if (b > need) need = b; };
    if (rows > 0 && H > 0) {
        const int R = rows < (1LL << 30) ? static_cast<int>(rows) : (1 << 30);
        auto colsum_bound = [&](long long N) { return 4 * (N > 6LL * 256 * num_sms() ? N : 6LL * 256 * num_sms()); };
        const int shapes[4][2] = {{3 * H, H}, {H, H}, {I, H}, {H, I}};
        for (const auto& sh : shapes) {
            if (sh[0] <= 0 || sh[1] <= 0) continue;
            const int splits = max_splits(gemm_tiles(sh[0], sh[1]), R);
            if (splits > 1) up(static_cast<long long>(splits) * sh[0] * sh[1] * 4);
        }
        long long last_tiles = -1;
        int splits = 1;
        for (int v = 16; v <= (vocab + 15) / 16 * 16; v += 16) {
            const long long t = gemm_tiles(v, H);
            if (t != last_tiles) { splits = max_splits(t, R); last_tiles = t; }
            if (splits > 1) up(static_cast<long long>(splits) * v * H * 4);
        }
        up(colsum_bound((vocab + 15) / 16 * 16));
        up(colsum_bound(I > 3 * H ? I : 3 * H));
        up(ln_bwd_det_bytes(R, H));
        up(embed_bwd_det_bytes(1, R, 0, H, -1));   // 3 items per row: at least as many as any split of `rows` into text and regions
    }
    return align256(need);
}

}  // namespace vb

extern "C" {
int64_t vb_deterministic_workspace_bytes(int64_t rows, int32_t hidden, int32_t inter, int32_t vocab, int32_t adam_chunks) {
    if (rows < 0 || hidden < 0 || inter < 0 || vocab < 0 || adam_chunks < 0 || (rows > 0 && hidden % 8 != 0)) {
        vb::set_error("vb_deterministic_workspace_bytes: bad shape (rows %lld, hidden %d, inter %d, vocab %d, adam_chunks %d)",
                      static_cast<long long>(rows), hidden, inter, vocab, adam_chunks);
        return -1;
    }
    return vb::deterministic_workspace_bytes(rows, hidden, inter, vocab, adam_chunks);
}
int vb_layer_fwd(const vb_layer_desc* d, const void* x_in, void* x_out, const vb_layer_acts* acts, void* stream) {
    return vb::layer_fwd(d, x_in, x_out, acts, static_cast<cudaStream_t>(stream));
}
int vb_layer_bwd(const vb_layer_desc* d, const void* x_in, const vb_layer_acts* acts, const void* dy, void* dx,
                 const vb_layer_grads* grads, const vb_layer_scratch* scratch, void* stream) {
    return vb::layer_bwd(d, x_in, acts, dy, dx, grads, scratch, static_cast<cudaStream_t>(stream));
}
int64_t vb_encoder_arena_layout(int32_t batch, int32_t seq, int32_t hidden, int32_t heads, int32_t inter, int32_t attn_dropout_on,
                                int64_t* offsets) {
    long long off[VB_ENCODER_ARENA_BUFFERS];
    const long long stride = vb::encoder_arena_layout(batch, seq, hidden, heads, inter, attn_dropout_on, off);
    if (offsets) for (int i = 0; i < VB_ENCODER_ARENA_BUFFERS; ++i) offsets[i] = off[i];
    return stride;
}
int vb_encoder_fwd(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* arena, void* stream) {
    return vb::encoder_fwd(descs, n_layers, x_in, arena, static_cast<cudaStream_t>(stream));
}
int vb_encoder_bwd(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* arena, const void* dy, void* dx,
                   const vb_layer_grads* grads, const vb_layer_scratch* scratch, void* stream) {
    return vb::encoder_bwd(descs, n_layers, x_in, arena, dy, dx, grads, scratch, static_cast<cudaStream_t>(stream));
}
int vb_encoder_attention_probs(const vb_layer_desc* descs, int32_t n_layers, void* arena, float* probs, void* stream) {
    return vb::encoder_attention_probs(descs, n_layers, arena, probs, static_cast<cudaStream_t>(stream));
}
int64_t vb_encoder_arena_layout_varlen(int32_t batch, int32_t max_seq, int32_t total, int32_t hidden, int32_t heads, int32_t inter,
                                       int32_t attn_dropout_on, int64_t* offsets) {
    if (batch <= 0 || max_seq <= 0 || total < 0) {
        vb::set_error("vb_encoder_arena_layout_varlen: bad shape (batch %d, max_seq %d, total %d)", batch, max_seq, total);
        return -1;
    }
    long long off[VB_ENCODER_ARENA_BUFFERS];
    const long long stride = vb::encoder_arena_layout(batch, max_seq, hidden, heads, inter, attn_dropout_on, off, total);
    if (offsets) for (int i = 0; i < VB_ENCODER_ARENA_BUFFERS; ++i) offsets[i] = off[i];
    return stride;
}
int vb_encoder_fwd_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total, const void* x_in,
                          void* arena, void* stream) {
    if (cu_seqlens == nullptr) { vb::set_error("vb_encoder_fwd_varlen: cu_seqlens is NULL"); return 2; }
    if (total <= 0) { vb::set_error("vb_encoder_fwd_varlen: total (%d) must be > 0", total); return 2; }
    const vb::LayerRows rows = {cu_seqlens, total};
    return vb::encoder_fwd(descs, n_layers, x_in, arena, static_cast<cudaStream_t>(stream), rows);
}
int64_t vb_encoder_infer_workspace(int32_t batch, int32_t seq, int32_t hidden, int32_t heads, int32_t inter, int32_t attn_dropout_on,
                                   int64_t packed_rows) {
    if (batch <= 0 || seq <= 0 || hidden <= 0 || heads <= 0 || inter <= 0 || packed_rows == 0 || packed_rows >= (1LL << 31)) {
        vb::set_error("vb_encoder_infer_workspace: bad shape (batch %d, seq %d, hidden %d, heads %d, inter %d, packed_rows %lld)", batch,
                      seq, hidden, heads, inter, static_cast<long long>(packed_rows));
        return -1;
    }
    return vb::infer_workspace_layout(batch, seq, hidden, heads, inter, attn_dropout_on, packed_rows, nullptr);
}
int vb_encoder_infer(const vb_layer_desc* descs, int32_t n_layers, const void* x_in, void* workspace, void* y_last, void* y_all,
                     float* probs, void* stream) {
    return vb::encoder_infer(descs, n_layers, x_in, workspace, y_last, y_all, probs, static_cast<cudaStream_t>(stream));
}
int vb_encoder_infer_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total, const void* x_in,
                            void* workspace, void* y_last, void* y_all, void* stream) {
    if (cu_seqlens == nullptr) { vb::set_error("vb_encoder_infer_varlen: cu_seqlens is NULL"); return 2; }
    if (total <= 0) { vb::set_error("vb_encoder_infer_varlen: total (%d) must be > 0", total); return 2; }
    const vb::LayerRows rows = {cu_seqlens, total};
    return vb::encoder_infer(descs, n_layers, x_in, workspace, y_last, y_all, nullptr, static_cast<cudaStream_t>(stream), rows);
}
int vb_encoder_bwd_varlen(const vb_layer_desc* descs, int32_t n_layers, const int32_t* cu_seqlens, int32_t total, const void* x_in,
                          void* arena, const void* dy, void* dx, const vb_layer_grads* grads, const vb_layer_scratch* scratch,
                          void* stream) {
    if (cu_seqlens == nullptr) { vb::set_error("vb_encoder_bwd_varlen: cu_seqlens is NULL"); return 2; }
    if (total <= 0) { vb::set_error("vb_encoder_bwd_varlen: total (%d) must be > 0", total); return 2; }
    const vb::LayerRows rows = {cu_seqlens, total};
    return vb::encoder_bwd(descs, n_layers, x_in, arena, dy, dx, grads, scratch, static_cast<cudaStream_t>(stream), rows);
}
int vb_embed_fwd(const vb_embed_desc* d, void* y, const vb_embed_acts* acts, void* stream) {
    return vb::embed_fwd_api(d, y, acts, static_cast<cudaStream_t>(stream));
}
int vb_embed_bwd(const vb_embed_desc* d, const vb_embed_acts* acts, const void* dy, const vb_embed_grads* g, void* stream) {
    return vb::embed_bwd_api(d, acts, dy, g, static_cast<cudaStream_t>(stream));
}
int vb_mask_bias(const int64_t* input_mask, const int64_t* image_mask, float* out, int32_t batch, int32_t text_len,
                 int32_t num_regions, void* stream) {
    return vb::mask_bias(reinterpret_cast<const long long*>(input_mask), reinterpret_cast<const long long*>(image_mask),
                         out, batch, text_len, num_regions, static_cast<cudaStream_t>(stream));
}
int vb_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream) {
    return vb::cast_f32_bf16(src, dst, n, static_cast<cudaStream_t>(stream));
}
int vb_cast_bf16_to_f32(const void* src, float* dst, int64_t n, void* stream) {
    return vb::cast_bf16_f32(src, dst, n, static_cast<cudaStream_t>(stream));
}
int vb_colsum_bf16(const void* x, int64_t ld, float* out, int32_t rows, int32_t cols, void* stream) {
    return vb::colsum(x, ld, out, rows, cols, static_cast<cudaStream_t>(stream));
}
}
