// vb_gemm.cu — the dense-contraction core of the VisualBERT encoder hot path on sm_90a.
//
// One warp-specialised kernel computes D[M,N] = epi(sum_k A(m,k) B(n,k)) in bf16 with fp32 accumulation,
// one 128 x BLOCK_N tile per CTA (BLOCK_N = 256, or 128 for narrow / ragged N):
//   warpgroup 0     TMA producer  (one elected thread: cp.async.bulk.tensor, 128B-swizzled 64-wide k-slabs,
//                                  4-stage mbarrier ring; after the last k-slab, the epilogue operand — residual /
//                                  gelu' / O — into the slots that drained first)
//   warpgroups 1-2  MMA + epilogue (wgmma.mma_async 64 x 256 x 16, or 64 x 128 x 16 on 128-wide tiles, from shared-memory
//                                  descriptors, fp32 accumulators in registers, 64 rows per warpgroup; bf16 outputs:
//                                  bias / dropout / residual / GELU / GELU' on the accumulator fragment, stmatrix into
//                                  the drained ring, a TMA store per 64 columns; fp32 outputs: the tile goes through
//                                  shared memory for red.add of split-K weight gradients)
//
// Replaces every nn.Linear on the path (reference modeling.py:232-234 Q/K/V, 271 attention output,
// 303 intermediate, 316 output, 1220 visual projection) together with the element-wise work that
// follows each of them (bias, dropout 272/317, residual add 273/318, gelu 304), and their autograd
// backward (input gradients use B "MN-major", weight gradients use A and B "MN-major").
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <vector>

#include "../../include/vbert_b200.h"
#include "vb_common.cuh"

namespace vb {

// ---------------------------------------------------------------------------------------------
// error + launch accounting (host)
// ---------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* get_error() { return g_err; }

// ---- deterministic reductions: thread-local like the error message (the autograd engine runs backward on its own thread) ----
static thread_local void* g_det_ptr = nullptr;
static thread_local long long g_det_bytes = 0;
DetWs det_ws() { return DetWs{g_det_ptr, g_det_bytes}; }
int det_require(long long need, const char* what) {
    VB_REQUIRE(g_det_ptr == nullptr || need <= g_det_bytes,
               "%s: deterministic mode needs %lld bytes of workspace, %lld are set (vb_deterministic_workspace_bytes)", what, need,
               g_det_bytes);
    return 0;
}
// ---- dropout seed offset in device memory: thread-local for the same reason ----
static thread_local const unsigned long long* g_drop_offset = nullptr;
const unsigned long long* drop_offset() { return g_drop_offset; }

// ---- live profiling -------------------------------------------------------------------------
struct ProfRec { cudaEvent_t e0, e1; int cat; double work; int launches; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;      // records in use
static std::vector<ProfRec> g_prof_pool; // recycled event pairs
static std::mutex g_prof_mu;

ProfScope::ProfScope(cudaStream_t s, int cat, double work, int launches) : slot(-1), st(s) {
    g_launches.fetch_add(launches);
    if (!g_prof_on) return;
    // an event recorded into a capturing stream becomes a graph node, not a timestamp this process can read back
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(s, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    ProfRec r;
    if (!g_prof_pool.empty()) { r = g_prof_pool.back(); g_prof_pool.pop_back(); }
    else { cudaEventCreate(&r.e0); cudaEventCreate(&r.e1); }
    r.cat = cat; r.work = work; r.launches = launches;
    cudaEventRecord(r.e0, st);
    g_prof.push_back(r);
    slot = static_cast<int>(g_prof.size()) - 1;
}
ProfScope::~ProfScope() {
    if (slot < 0) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    cudaEventRecord(g_prof[slot].e1, st);
}

// ---------------------------------------------------------------------------------------------
// tile configuration
// ---------------------------------------------------------------------------------------------
constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle atom row
constexpr int WGMMA_K = 16;
constexpr int kStages = 4;
constexpr int kEpiWarps = 8;                    // the two MMA warpgroups
constexpr int kThreads = 128 + kEpiWarps * 32;  // 384
constexpr int kAtomBytes = 64 * BLOCK_K * 2;    // one 64(MN) x 64(K) bf16 swizzle atom = 8 KB

template <int BLOCK_N>
struct Cfg {
    static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
    static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    // fp32 outputs: the accumulator tile goes through shared memory over the drained operand ring; +4 floats per row keeps the
    // row-per-lane reads of that epilogue free of bank conflicts
    static constexpr int ACC_LD = BLOCK_N + 4;
    static constexpr int RING_BYTES = kStages * STAGE_BYTES > BLOCK_M * ACC_LD * 4 ? kStages * STAGE_BYTES : BLOCK_M * ACC_LD * 4;
    // bf16 outputs: the ring is reused in 16 KB pieces (128 rows x 64 columns of bf16, 128B-swizzled like the k-slabs), taken
    // in the order in which the slots drain (see piece_addr): pieces [0, OPND) receive the epilogue operand while the last
    // k-blocks still compute, pieces [OPND, OPND + 2 OPND) stage the one or two bf16 outputs for the TMA stores
    static constexpr int PIECE = 16384;
    static constexpr int PIECES_PER_SLOT = STAGE_BYTES / PIECE;
    static constexpr int OPND = BLOCK_N / 64;
    static constexpr int OPND_SLOTS = (OPND + PIECES_PER_SLOT - 1) / PIECES_PER_SLOT;
    static_assert(STAGE_BYTES % PIECE == 0 && 3 * OPND <= kStages * PIECES_PER_SLOT, "operand + two output tiles fit the ring");
    static constexpr int BAR_OFF = RING_BYTES;
    static constexpr int NUM_BARS = 2 * kStages + 1;   // full / empty per slot, + the epilogue operand
    static constexpr int BIAS_OFF = (BAR_OFF + NUM_BARS * 8 + 15) / 16 * 16;
    static constexpr int SMEM_BYTES = BIAS_OFF + BLOCK_N * 4 + 1024;  // +1024: manual 1 KB alignment
    static_assert(SMEM_BYTES <= 227 * 1024, "shared memory per block");
};

struct GemmParams {
    int M, N, K;
    int splits;
    void* D; long long ldd;
    const float* bias;
    const bf16* addend; long long ld_add;
    int epilogue;
    const bf16* aux_in;
    bf16* aux_out; long long ld_aux;
    float drop_scale;        // 256/(256-n), 0 => dropout off
    unsigned drop_thresh16;  // n = round(p * 256): 8-bit keep threshold (see dropout_quantise)
    unsigned long long drop_seed;
    unsigned drop_stream;
    int m_fast;              // tile order: m-blocks run faster than n-blocks (see decode_tile)
    union {
        float* delta_out;        // EPI_DELTA: fp32 [rows / delta_seq][N / 64][delta_seq]
        const unsigned long long* drop_offset;   // EPI_GENERIC_OFF: device offset added to drop_seed (a dropout GEMM has no delta)
    };
    int delta_seq;
};
bool gemm_gp_tiled_ok(int M, int N);
bool gemm_delta_ok(int M, int N);

struct TileCoord {
    int m_blk, n_blk, kb_begin, kb_end;
};
// Tile order: the split index runs slowest, so that the CTAs in flight at any time work on one or two k-ranges; within a split
// the dimension with FEWER blocks runs fastest (m_fast: there are fewer m-blocks), so that those CTAs share the slabs of the
// operand that spans the dimension with MORE blocks — the big one, which must not be fetched from DRAM once per block of the
// other dimension (FFN-down weight gradient: M = 768, N = 3072, B = gelu(u) is several times the L2).
__device__ __forceinline__ TileCoord decode_tile(int t, int n_blocks, int splits, int k_blocks, int m_blocks, bool m_fast) {
    TileCoord c;
    const int tiles = m_blocks * n_blocks;
    const int split = t / tiles;
    const int mn = t - split * tiles;
    if (m_fast) {
        c.m_blk = mn % m_blocks;
        c.n_blk = mn / m_blocks;
    } else {
        c.n_blk = mn % n_blocks;
        c.m_blk = mn / n_blocks;
    }
    c.kb_begin = static_cast<int>(static_cast<long long>(split) * k_blocks / splits);
    c.kb_end = static_cast<int>(static_cast<long long>(split + 1) * k_blocks / splits);
    return c;
}

// EPI selects the epilogue at COMPILE time: the generic form (every option a run-time branch) is several times larger than one
// specialised path, and instruction-cache misses then stall the epilogue. A specialised kernel carries only its path.
// _T: gelu'(u) is kept in the TILE-NATIVE layout (vb_gemm_args.gp_tiled, include/vbert_b200.h): the 64 KB of one tile are
// contiguous, so the GELU epilogue stores them and the backward GEMM's epilogue loads them with one bulk copy per 16 KB.
// EPI_DELTA: plain bf16 store plus the attention backward's D[b, head, s] = sum_d dO[row, head, d] * O[row, head, d] (vb_gemm_args.delta_*):
// the GEMM that PRODUCES dO (input gradient of attention.output.dense) has whole heads in each tile; O is loaded like a residual
// operand, and each row's dot products are taken in column order from the staged dO and O once the tile is staged.
// EPI_GELU_ONLY (VB_EPI_GELU_FWD of the ABI): D = gelu(u) and nothing else — the forward-only FFN-up GEMM, with the gelu of the
// two-tensor epilogues.
// EPI_SLAB (fp32 output, deterministic mode): split s STORES its partial tile to slab s of the workspace, D = slab base with
// ldd = N, slab s at D + s * M * N, no bias; splitk_reduce_kernel then adds bias + the slabs in split order into the real D.
enum { EPI_GENERIC = 0, EPI_BIAS = 1, EPI_RESID = 2, EPI_DROP_RESID = 3, EPI_GELU_FWD = 4, EPI_DGELU_BWD = 5, EPI_GELU_FWD_T = 6,
       EPI_DGELU_BWD_T = 7, EPI_DELTA = 8, EPI_GELU_ONLY = 9, EPI_SLAB = 10, EPI_GENERIC_OFF = 11 };
// EPI_GENERIC_OFF: the generic epilogue with the dropout seed p.drop_seed + *p.drop_offset, read from device memory when the
// epilogue runs (vb_set_dropout_offset); a call with dropout takes it whenever an offset is set, so no other kernel reads it.
__host__ __device__ constexpr bool epi_is_generic(int e) { return e == EPI_GENERIC || e == EPI_GENERIC_OFF; }
__host__ __device__ constexpr bool epi_is_gelu(int e) { return e == EPI_GELU_FWD || e == EPI_GELU_FWD_T; }
__host__ __device__ constexpr bool epi_is_dgelu(int e) { return e == EPI_DGELU_BWD || e == EPI_DGELU_BWD_T; }
// the epilogue reads a [128, BLOCK_N] bf16 operand (residual, gelu'(u) or O): compile-time "may", run-time "does"
__host__ __device__ constexpr bool epi_may_read(int e) {
    return e == EPI_RESID || e == EPI_DROP_RESID || epi_is_dgelu(e) || e == EPI_DELTA || epi_is_generic(e);
}
__device__ __forceinline__ bool epi_reads(int e, const GemmParams& p) {
    return e == EPI_RESID || e == EPI_DROP_RESID || epi_is_dgelu(e) || e == EPI_DELTA ||
           (epi_is_generic(e) && (p.addend != nullptr || p.epilogue == VB_EPI_DGELU));
}

template <int BLOCK_N, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BLOCK_N / 2], uint64_t ad, uint64_t bd, uint32_t accumulate) {
    if constexpr (BLOCK_N == 256) wgmma_m64n256k16<TA, TB>(acc, ad, bd, accumulate);
    else wgmma_m64n128k16<TA, TB>(acc, ad, bd, accumulate);
}

// byte offset of element (row, col) of a 128 x 256 tile in the tile-native gelu'(u) layout (include/vbert_b200.h): eight 8 KB
// blocks (column half, 32-row group), in each eight 1 KB blocks of 16 columns, row r of the 32 at + 32 r
__device__ __forceinline__ uint32_t tn_byte(int row, int col) {
    return ((((col >> 7) * 4 + (row >> 5)) * 8 + ((col & 127) >> 4)) * 512 + (row & 31) * 16 + (col & 15)) * 2;
}

template <bool A_MN, bool B_MN, int BLOCK_N, bool OUT_F32, int EPI = EPI_GENERIC>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p,
                  const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmE) {
    using C = Cfg<BLOCK_N>;
    static_assert(BLOCK_N == 128 || BLOCK_N == 256, "64 x 128 / 64 x 256 wgmma tiles");
    static_assert(!(EPI == EPI_GELU_FWD_T || EPI == EPI_DGELU_BWD_T) || BLOCK_N == 256, "tile-native gelu' is defined on 256-wide tiles");
    static_assert(!(EPI == EPI_DELTA) || BLOCK_N == 256, "EPI_DELTA: four whole heads per tile");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1 KB alignment
    uint8_t* smem = smem_raw + (base - raw);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    auto a_tile = [&](int s) { return base + s * C::STAGE_BYTES; };
    auto b_tile = [&](int s) { return base + s * C::STAGE_BYTES + C::A_BYTES; };
    auto full_bar = [&](int s) { return base + C::BAR_OFF + 8 * s; };
    auto empty_bar = [&](int s) { return base + C::BAR_OFF + 8 * (kStages + s); };
    const uint32_t opnd_bar = base + C::BAR_OFF + 8 * (2 * kStages);

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 2);   // one arrival per MMA warpgroup
        }
        mbar_init(opnd_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();  // everything above is on-chip set-up; operands of the previous kernel are read only from here on

    const int m_blocks = (p.M + BLOCK_M - 1) / BLOCK_M;
    const int n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
    const int k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
    const TileCoord tc = decode_tile(blockIdx.x, n_blocks, p.splits, k_blocks, m_blocks, p.m_fast != 0);
    // piece k of the ring (bf16 outputs): the slots in the order in which they drain — the slot the next k-block would have
    // used first (its last k-block is the oldest), PIECES_PER_SLOT pieces per slot
    const int n_kb = tc.kb_end - tc.kb_begin;
    auto piece_addr = [&](int k) {
        return base + ((n_kb + k / C::PIECES_PER_SLOT) % kStages) * C::STAGE_BYTES + (k % C::PIECES_PER_SLOT) * C::PIECE;
    };
    const long long tn_tile = ((static_cast<long long>(tc.m_blk >> 1) * n_blocks + tc.n_blk) * 2 + (tc.m_blk & 1)) * (BLOCK_M * BLOCK_N);

    if (warp < 4) {
        reg_dec<40>();
        if (warp == 0) {
            // ---------------- TMA producer (converged warp, one elected lane issues) ----------------
            int stage = 0;
            uint32_t phase = 0;
            for (int kb = tc.kb_begin; kb < tc.kb_end; ++kb) {
                mbar_wait(empty_bar(stage), phase ^ 1u);
                if (elect_one()) {
                    mbar_arrive_expect_tx(full_bar(stage), C::STAGE_BYTES);
                    if constexpr (!A_MN) {
                        tma_load_2d(a_tile(stage), &tmA, full_bar(stage), kb * BLOCK_K, tc.m_blk * BLOCK_M);
                    } else {
#pragma unroll
                        for (int i = 0; i < BLOCK_M / 64; ++i)
                            tma_load_2d(a_tile(stage) + i * kAtomBytes, &tmA, full_bar(stage), tc.m_blk * BLOCK_M + i * 64, kb * BLOCK_K);
                    }
                    if constexpr (!B_MN) {
                        tma_load_2d(b_tile(stage), &tmB, full_bar(stage), kb * BLOCK_K, tc.n_blk * BLOCK_N);
                    } else {
#pragma unroll
                        for (int i = 0; i < BLOCK_N / 64; ++i)
                            tma_load_2d(b_tile(stage) + i * kAtomBytes, &tmB, full_bar(stage), tc.n_blk * BLOCK_N + i * 64, kb * BLOCK_K);
                    }
                }
                __syncwarp();
                if (++stage == kStages) { stage = 0; phase ^= 1u; }
            }
            if constexpr (!OUT_F32 && epi_may_read(EPI)) {
                if (epi_reads(EPI, p)) {
                    // the epilogue operand goes into the oldest slots as soon as their last k-blocks have retired, while the
                    // MMAs of the newest ones still run: wait for them as for the next k-blocks
                    for (int t = 0; t < C::OPND_SLOTS; ++t) {
                        mbar_wait(empty_bar(stage), phase ^ 1u);
                        if (++stage == kStages) { stage = 0; phase ^= 1u; }
                    }
                    if (elect_one()) {
                        mbar_arrive_expect_tx(opnd_bar, C::OPND * C::PIECE);
                        if (EPI == EPI_DGELU_BWD_T) {
                            const uint8_t* src = reinterpret_cast<const uint8_t*>(p.aux_in) + tn_tile * 2;
#pragma unroll
                            for (int k = 0; k < C::OPND; ++k) bulk_load(piece_addr(k), src + k * C::PIECE, C::PIECE, opnd_bar);
                        } else {
                            tma_prefetch_desc(&tmE);
#pragma unroll
                            for (int k = 0; k < C::OPND; ++k)
                                tma_load_2d(piece_addr(k), &tmE, opnd_bar, tc.n_blk * BLOCK_N + 64 * k, tc.m_blk * BLOCK_M);
                        }
                    }
                    __syncwarp();
                }
            }
        }
        return;
    }
    reg_inc<232>();

    // ---------------- MMA warpgroups: rows 64 wg .. 64 wg + 63 of the tile, all BLOCK_N columns ----------------
    const int wg = (warp >> 2) - 1;
    const int et = threadIdx.x - 128;  // 0..255 among the MMA / epilogue threads
    float* sbias = reinterpret_cast<float*>(smem + C::BIAS_OFF);
    const bool has_bias = p.bias != nullptr;
    if (has_bias) {   // with split-K the bias belongs to the whole sum: only split 0 adds it, the other splits stage zeros
        const bool mine = tc.kb_begin == 0;
        for (int i = et; i < BLOCK_N; i += kEpiWarps * 32) {
            const int col = tc.n_blk * BLOCK_N + i;
            sbias[i] = (mine && col < p.N) ? __ldg(p.bias + col) : 0.f;
        }
    }
    // K-major: advance 16 elements (32 B) inside the swizzle row; MN-major: 16 k-rows (2 KB)
    constexpr uint32_t a_kstep = A_MN ? WGMMA_K * 128 : WGMMA_K * 2;
    constexpr uint32_t b_kstep = B_MN ? WGMMA_K * 128 : WGMMA_K * 2;
    // fragment (wgmma_m64n128k16 / wgmma_m64n256k16): acc[4 j + 2 i + c] = tile[64 wg + 16 (warp % 4) + lane / 4 + 8 i][8 j + 2 (lane % 4) + c]
    float acc[BLOCK_N / 2];
    {
        int stage = 0, prev = 0;
        uint32_t phase = 0;
        for (int kb = tc.kb_begin; kb < tc.kb_end; ++kb) {
            mbar_wait(full_bar(stage), phase);
            // this warpgroup's 64 rows of A: 64 K-major rows or one 64-wide MN-major atom = 8 KB further in both layouts
            const uint32_t a0 = a_tile(stage) + wg * 8192, b0 = b_tile(stage);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / WGMMA_K; ++k)
                wgmma_tile<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, wgmma_desc_sw128(a0 + k * a_kstep, kAtomBytes, 1024),
                                                              wgmma_desc_sw128(b0 + k * b_kstep, kAtomBytes, 1024),
                                                              (kb > tc.kb_begin || k > 0) ? 1u : 0u);
            wgmma_commit();
            // the MMAs of the previous k-block have retired: its slot may be refilled
            wgmma_wait<1>();
            if (kb > tc.kb_begin && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar(prev));
            prev = stage;
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
    }
    // both warpgroups' MMAs have retired (and with them every read of the ring): the ring may be overwritten
    named_bar_sync(1, kEpiWarps * 32);

    if constexpr (OUT_F32) {
        // ---------------- fp32 epilogue: split-K red.add or a deterministic slab store ----------------
        // The tile goes through shared memory so that a thread owns 16-column pieces of one row: lane l of epilogue warp ew
        // takes chunk l / RPI of row RPI k + l % RPI of rows 32 (ew % 4) .. + 31, column half ew / 4, so that one warp access
        // covers whole half-rows.
        float* sacc = reinterpret_cast<float*>(smem);
        {
            const int r0 = wg * 64 + ((warp & 3) << 4) + (lane >> 2);
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i)
                    *reinterpret_cast<float2*>(sacc + (r0 + 8 * i) * C::ACC_LD + j * 8 + 2 * (lane & 3)) =
                        make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
        }
        named_bar_sync(1, kEpiWarps * 32);
        const int ew = warp - 4;
        const int q = ew & 3, half = ew >> 2;
        constexpr int NCH = BLOCK_N / 2 / 16;
        constexpr int RPI = 32 / NCH;
#pragma unroll
        for (int k = 0; k < NCH; ++k) {
            const int lrow = q * 32 + RPI * k + lane % RPI, cc = half * (BLOCK_N / 2) + (lane / RPI) * 16;   // in the tile
            const int row = tc.m_blk * BLOCK_M + lrow;
            const int col = tc.n_blk * BLOCK_N + cc;
            if (row < p.M && col < p.N) {
                float x[16];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float4 v = *reinterpret_cast<const float4*>(sacc + lrow * C::ACC_LD + cc + 4 * i);
                    x[4 * i] = v.x; x[4 * i + 1] = v.y; x[4 * i + 2] = v.z; x[4 * i + 3] = v.w;
                }
                if constexpr (EPI == EPI_SLAB) {
                    float* d = reinterpret_cast<float*>(p.D) + (static_cast<long long>(blockIdx.x / (m_blocks * n_blocks)) * p.M + row) * p.ldd + col;
#pragma unroll
                    for (int i = 0; i < 4; ++i) *reinterpret_cast<float4*>(d + 4 * i) = make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
                } else {
                    if (has_bias) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const float4 b = *reinterpret_cast<const float4*>(sbias + cc + 4 * i);
                            x[4 * i] += b.x; x[4 * i + 1] += b.y; x[4 * i + 2] += b.z; x[4 * i + 3] += b.w;
                        }
                    }
                    float* d = reinterpret_cast<float*>(p.D) + static_cast<long long>(row) * p.ldd + col;
#pragma unroll
                    for (int i = 0; i < 4; ++i) red_add_v4_f32(d + 4 * i, x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
                }
            }
        }
    } else {
        // ---------------- bf16 epilogue in the accumulator fragment ----------------
        // Per element, in this order: + bias, dropout, + residual, then GELU (two outputs) / x gelu'(u) / gelu only. The operand
        // comes from shared memory (loaded by the producer warp) and the results are staged there, both with ldmatrix /
        // stmatrix on 8 x 8 blocks; each warpgroup then stores its 64 rows with TMA (out-of-bounds rows and columns clipped).
        constexpr bool kGeneric = epi_is_generic(EPI);
        constexpr bool kTwoOut = epi_is_gelu(EPI) || kGeneric;    // generic: GELU at run time
        const bool two_out = epi_is_gelu(EPI) || (kGeneric && p.epilogue == VB_EPI_GELU);
        const bool reads = epi_may_read(EPI) && epi_reads(EPI, p);
        const bool is_dgelu = epi_is_dgelu(EPI) || (kGeneric && p.epilogue == VB_EPI_DGELU);
        const bool add = EPI == EPI_RESID || EPI == EPI_DROP_RESID || (kGeneric && p.addend != nullptr);
        const bool drop = EPI == EPI_DROP_RESID || (kGeneric && p.drop_scale != 0.0f);
        const int w4 = warp & 3, qd = lane & 3;
        const int frow0 = 64 * wg + 16 * w4 + (lane >> 2);            // tile row of acc[.. + 0], +8 for acc[.. + 2]
        const int mrow = 64 * wg + 16 * w4 + ((lane >> 3) & 1) * 8 + (lane & 7);   // row this lane addresses in ldmatrix / stmatrix
        const int mj = lane >> 4;                                      // ... and its 8-column block within a pair
        // row-major tiles: 64-column pieces, row r at + 128 r, its 16-byte blocks permuted by r % 8 (the TMA 128B swizzle);
        // piece p0 + col / 64 holds the columns of `col`
        auto rm_addr = [&](int p0, int col) {
            return piece_addr(p0 + (col >> 6)) + mrow * 128 + ((((col & 63) >> 3) ^ (mrow & 7)) << 4);
        };
        auto tn_addr = [&](int pbase, int col) {   // tile-native staging / operand
            const uint32_t o = tn_byte(mrow, col);
            return piece_addr(pbase + (o >> 14)) + (o & (C::PIECE - 1));
        };

        // dropout keep words: lane qd draws the word of 8-column group 4 t + qd of its two rows; the quad exchanges them below
        constexpr int KW = BLOCK_N / 128;   // words per row: 4 groups (one byte each) of the lane's BLOCK_N / 32
        uint32_t kw[2][KW];
        if (drop) {
            const uint32_t key0 = dropout_key(EPI == EPI_GENERIC_OFF ? p.drop_seed + *p.drop_offset : p.drop_seed, p.drop_stream);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const unsigned long long e0 =
                    (static_cast<unsigned long long>(tc.m_blk * BLOCK_M + frow0 + 8 * i) * static_cast<unsigned>(p.N) + tc.n_blk * BLOCK_N) >> 3;
#pragma unroll
                for (int s = 0; s < KW; ++s) {
                    uint32_t w = 0;
#pragma unroll
                    for (int b = 0; b < 4; ++b) w |= dropout_keep8_key(key0, e0 + 4 * (4 * s + b) + qd, p.drop_thresh16) << (8 * b);
                    kw[i][s] = w;
                }
            }
        }
        // the words of the quad's four lanes: kq[i][s][q] = kw[i][s] of lane q
        uint32_t kq[2][KW][4];
        if (drop) {
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int s = 0; s < KW; ++s)
#pragma unroll
                    for (int q = 0; q < 4; ++q) kq[i][s][q] = __shfl_sync(0xffffffffu, kw[i][s], (lane & ~3) | q);
        }
        if (reads) mbar_wait(opnd_bar, 0);

#pragma unroll
        for (int jp = 0; jp < BLOCK_N / 16; ++jp) {
            // registers k = 0..3 of this pair: 8-column block j = 2 jp + k / 2, row frow0 + 8 (k % 2) = acc[8 jp + 2 k], +1
            float* x = acc + 8 * jp;
            const int mcol = 16 * jp + 8 * mj;   // the column block this lane addresses
            if (has_bias) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float2 b = *reinterpret_cast<const float2*>(sbias + 8 * (2 * jp + k / 2) + 2 * qd);
                    x[2 * k] += b.x; x[2 * k + 1] += b.y;
                }
            }
            if (drop) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int j = 2 * jp + k / 2;   // group j was drawn by lane j % 4 of the quad: byte (j / 4) % 4 of its word j / 16
                    const uint32_t keep = kq[k % 2][j / 16][j & 3] >> (8 * ((j >> 2) & 3) + 2 * qd);
                    x[2 * k] = (keep & 1u) ? x[2 * k] * p.drop_scale : 0.0f;
                    x[2 * k + 1] = (keep & 2u) ? x[2 * k + 1] * p.drop_scale : 0.0f;
                }
            }
            uint32_t e[4] = {0u, 0u, 0u, 0u};
            if (reads) {
                if (EPI == EPI_DGELU_BWD_T) ldmatrix_x4(tn_addr(0, mcol), e);
                else ldmatrix_x4(rm_addr(0, mcol), e);
            }
            if (add) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float2 t = unpack_bf16x2(e[k]);
                    x[2 * k] += t.x;
                    x[2 * k + 1] += t.y;
                }
            }
            uint32_t o0[4], o1[4];
            if (EPI == EPI_GELU_ONLY) {
                // D <- gelu(u): the value the GELU epilogue below sends to aux_out, from the same function; its derivative is dropped
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    float gp;
                    gelu_fwd_bwd(x[k], x[k], gp);
                }
            } else if (kTwoOut && two_out) {
                // aux_out <- gelu(u) (operand of the next GEMM), D <- gelu'(u) (all the backward needs of u)
                float gp[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) gelu_fwd_bwd(x[k], x[k], gp[k]);
#pragma unroll
                for (int k = 0; k < 4; ++k) o1[k] = pack_bf16x2(gp[2 * k], gp[2 * k + 1]);
            } else if (is_dgelu) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float2 t = unpack_bf16x2(e[k]);
                    x[2 * k] *= t.x;
                    x[2 * k + 1] *= t.y;
                }
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) o0[k] = pack_bf16x2(x[2 * k], x[2 * k + 1]);
            if (kTwoOut && two_out) {
                // gelu'(u) -> D (tile-native or row-major), gelu(u) -> aux_out (row-major)
                stmatrix_x4(EPI == EPI_GELU_FWD_T ? tn_addr(C::OPND, mcol) : rm_addr(C::OPND, mcol), o1);
                stmatrix_x4(rm_addr(2 * C::OPND, mcol), o0);
            } else {
                stmatrix_x4(rm_addr(C::OPND, mcol), o0);
            }
            if ((jp & 3) == 3) {
                // 64 columns of this warpgroup's 64 rows are staged: one thread stores them while the others go on (the
                // generic proxy's writes made visible to TMA first)
                fence_proxy_async_smem();
                named_bar_sync(2 + wg, 128);
                if ((threadIdx.x & 127) == 0) {
                    const int b = jp >> 2, gcol = tc.n_blk * BLOCK_N + 64 * b, grow = tc.m_blk * BLOCK_M + 64 * wg;
                    if (EPI == EPI_GELU_FWD_T) {
                        // column half h of rows 64 wg .. + 63 is the 16 KB piece 2 h + wg of the tile's 64 KB
                        if ((jp & 7) == 7) {
                            const int pc = 2 * (jp >> 3) + wg;
                            bulk_store(reinterpret_cast<uint8_t*>(p.D) + tn_tile * 2 + pc * C::PIECE, piece_addr(C::OPND + pc), C::PIECE);
                        }
                        tma_store_2d(&tmX, piece_addr(2 * C::OPND + b) + wg * 8192, gcol, grow);
                    } else {
                        tma_store_2d(&tmD, piece_addr(C::OPND + b) + wg * 8192, gcol, grow);
                        if (kTwoOut && two_out) tma_store_2d(&tmX, piece_addr(2 * C::OPND + b) + wg * 8192, gcol, grow);
                    }
                    bulk_commit();
                }
            }
        }
        if constexpr (EPI == EPI_DELTA) {
            // D = rowsum(dO * O) per head from the staged, ROUNDED dO (what the attention kernel will read) and O, both in
            // shared memory: thread t of the warpgroup sums heads 2 (t / 64), +1 of row t % 64, each in column order
            const int t = threadIdx.x & 127, r = 64 * wg + (t & 63), row = tc.m_blk * BLOCK_M + r;
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int h = 2 * (t >> 6) + hh;   // head h of the tile = 64-column piece h
                float sum = 0.f;
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const uint32_t off = r * 128 + ((c ^ (r & 7)) << 4);
                    const uint4 dv = *reinterpret_cast<const uint4*>(smem + (piece_addr(C::OPND + h) - base) + off);
                    const uint4 ov = *reinterpret_cast<const uint4*>(smem + (piece_addr(h) - base) + off);
                    const uint32_t du[4] = {dv.x, dv.y, dv.z, dv.w}, ou[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float2 x = unpack_bf16x2(du[i]), y = unpack_bf16x2(ou[i]);
                        sum = fmaf(x.x, y.x, fmaf(x.y, y.y, sum));
                    }
                }
                const int c4 = tc.n_blk * BLOCK_N + 64 * h;
                if (row < p.M && c4 < p.N) {
                    const int bi = row / p.delta_seq, si = row - bi * p.delta_seq;
                    p.delta_out[(static_cast<long long>(bi) * (p.N >> 6) + (c4 >> 6)) * p.delta_seq + si] = sum;
                }
            }
        }
        if ((threadIdx.x & 127) == 0) bulk_wait_read0();   // the shared memory stays valid until TMA has read it; the global writes drain after exit
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(sym);
    }
    return fn;
}

// Tensor-map cache: a training step encodes ~1000 descriptors (2 per GEMM, 3-4 per attention call), each a driver call of
// 1-2 us on the launch path; with the activation arena of vb_encoder_fwd/bwd the same (pointer, shape) tuples recur every
// step, so the encoded 128-byte maps are memoised per thread (no locks on the launch path; direct-mapped, 4096 slots).
struct TmapKey {
    const void* ptr; uint64_t d0, d1, d2, s0, s1; uint32_t b0, b1, b2, rank; int dev;
    bool operator==(const TmapKey& o) const {
        return ptr == o.ptr && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && s0 == o.s0 && s1 == o.s1 && b0 == o.b0 && b1 == o.b1 && b2 == o.b2 &&
               rank == o.rank && dev == o.dev;
    }
};
struct TmapSlot { TmapKey key; CUtensorMap map; bool used; };
constexpr int kTmapSlots = 4096;
static thread_local std::vector<TmapSlot>* g_tmap_cache = nullptr;

static int encode_tmap_cached(CUtensorMap* m, const void* ptr, uint32_t rank, const cuuint64_t* dims, const cuuint64_t* strides,
                              const cuuint32_t* box) {
    TmapKey k;
    memset(&k, 0, sizeof(k));
    k.ptr = ptr; k.rank = rank; k.dev = current_device();
    k.d0 = dims[0]; k.d1 = dims[1]; k.d2 = rank > 2 ? dims[2] : 1;
    k.s0 = strides[0]; k.s1 = rank > 2 ? strides[1] : 0;
    k.b0 = box[0]; k.b1 = box[1]; k.b2 = rank > 2 ? box[2] : 1;
    uint64_t h = reinterpret_cast<uintptr_t>(ptr) * 0x9E3779B97F4A7C15ull;
    h ^= (k.d0 * 31 + k.d1) * 0xBF58476D1CE4E5B9ull + k.d2 * 1315423911ull + k.s0 * 2654435761ull + k.s1 * 40503ull;
    h ^= (static_cast<uint64_t>(k.b1) << 20) ^ (static_cast<uint64_t>(k.b0) << 8) ^ k.b2 ^ (static_cast<uint64_t>(k.dev) << 40);
    h ^= h >> 29;
    if (g_tmap_cache == nullptr) { g_tmap_cache = new std::vector<TmapSlot>(kTmapSlots); for (auto& sl : *g_tmap_cache) sl.used = false; }
    TmapSlot& sl = (*g_tmap_cache)[h & (kTmapSlots - 1)];
    if (sl.used && sl.key == k) { *m = sl.map; return 0; }
    EncodeTiledFn fn = get_encode_fn();
    VB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled unavailable (driver too old / no GPU?)");
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    VB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (rank %u) failed with CUresult %d", rank, static_cast<int>(r));
    sl.key = k; sl.map = *m; sl.used = true;
    return 0;
}

// 2-D bf16 tensor map: `inner` contiguous elements, `outer` rows of stride ld elements;
// box = 64 x box_outer, 128-byte swizzle, out-of-bounds reads return zero.
int make_tmap_bf16(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                   uint32_t box_outer) {
    VB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA operand not 16-byte aligned");
    VB_REQUIRE((ld_elems * 2) % 16 == 0, "TMA operand row stride must be a multiple of 8 elements");
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {ld_elems * 2};
    cuuint32_t box[2] = {64, box_outer};
    return encode_tmap_cached(m, ptr, 2, dims, strides, box);
}

int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev < 0 || dev >= kMaxDevices) ? 0 : dev;
}

int num_sms() {
    static int n[kMaxDevices] = {0};
    const int dev = current_device();
    if (n[dev] == 0) {
        int v = 0;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        n[dev] = v > 0 ? v : 132;
    }
    return n[dev];
}

// the tensor maps of one call: A and B (k-slab loads), and for bf16 outputs D and aux_out (64 x 64 stores of a warpgroup's rows)
// and the epilogue operand (64-column x 128-row loads); maps a call does not use stay zero
struct GemmMaps { CUtensorMap a, b, d, x, e; };

template <bool A_MN, bool B_MN, int BLOCK_N, bool OUT_F32, int EPI = EPI_GENERIC>
static int launch(const GemmMaps& m, const GemmParams& p, cudaStream_t st) {
    using C = Cfg<BLOCK_N>;
    auto kern = gemm_wgmma_kernel<A_MN, B_MN, BLOCK_N, OUT_F32, EPI>;
    static int configured[kMaxDevices] = {0};
    VB_CHECK_CUDA(ensure_dyn_smem(kern, C::SMEM_BYTES, configured));
    const long long tiles = static_cast<long long>((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N) * p.splits;
    VB_REQUIRE(tiles < (1LL << 31), "vb_gemm: too many tiles");
    {
        ProfScope ps(st, OUT_F32 ? PROF_GEMM_WGRAD : (B_MN ? PROF_GEMM_DGRAD : PROF_GEMM_FWD), 2.0 * p.M * p.N * p.K, 1);
        VB_CHECK_CUDA(launch_pdl(kern, dim3(static_cast<unsigned>(tiles)), dim3(kThreads), C::SMEM_BYTES, st, m.a, m.b, p, m.d, m.x, m.e));
    }
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// Split-K factor of an fp32 (accumulating) output, from the shape: the k-range is cut into `splits` equal parts so that the
// tiles * splits CTAs fill whole waves of one CTA per SM. It minimises the time of the busiest SM in k-blocks, waves * (k-blocks
// per split + kCtaCost), where kCtaCost stands for what every CTA pays besides its main loop (launch, first TMA round trip,
// red.add of its partial tile); the smallest such factor wins.
int wgrad_splits(long long tiles, int k_blocks) {
    constexpr int kCtaCost = 4;
    const long long sms = num_sms();
    int best = 1;
    long long best_cost = -1;
    for (int s = 1; s <= k_blocks && s <= 32; ++s) {
        const long long cost = (tiles * s + sms - 1) / sms * ((k_blocks + s - 1) / s + kCtaCost);
        if (best_cost < 0 || cost < best_cost) { best = s; best_cost = cost; }
    }
    return best;
}

// D[M, N] += bias + sum_s slab[s] (fp32, slab s at slab + s * M * N), four columns per thread, the splits added in order
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ slab, int splits, int M, int N, const float* __restrict__ bias, float* __restrict__ D,
                     long long ldd) {
    const long long n4 = static_cast<long long>(M) * N / 4, plane = static_cast<long long>(M) * N;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long e = 4 * i;
        const int row = static_cast<int>(e / N), col = static_cast<int>(e - static_cast<long long>(row) * N);
        float4 a = *reinterpret_cast<const float4*>(slab + e);
        if (bias != nullptr) { a.x += bias[col]; a.y += bias[col + 1]; a.z += bias[col + 2]; a.w += bias[col + 3]; }
        for (int s = 1; s < splits; ++s) {
            const float4 b = *reinterpret_cast<const float4*>(slab + s * plane + e);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        float4* d = reinterpret_cast<float4*>(D + static_cast<long long>(row) * ldd + col);
        float4 o = *d;
        o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w;
        *d = o;
    }
}

// BLOCK_N of a call: 256 unless N is small or padding N up to a multiple of 256 wastes more than 1/8 of the columns
static bool use_bn256(int N) { return N >= 256 && ((N + 255) / 256 * 256 - N) * 8 <= N; }
long long gemm_tiles(int M, int N) {
    const bool bn256 = use_bn256(N);
    return static_cast<long long>((M + BLOCK_M - 1) / BLOCK_M) * ((N + (bn256 ? 255 : 127)) / (bn256 ? 256 : 128));
}
int gemm_k_blocks(int K) { return (K + BLOCK_K - 1) / BLOCK_K; }

bool gemm_delta_ok(int M, int N) {
    const int n_pad256 = (N + 255) / 256 * 256;
    return M >= 256 && N >= 256 && N % 64 == 0 && (n_pad256 - N) * 8 <= N;
}
bool gemm_gp_tiled_ok(int M, int N) {
    return M >= 256 && M % 256 == 0 && N % 256 == 0;
}

int gemm(const vb_gemm_args& a, cudaStream_t st) {
    VB_REQUIRE(a.M > 0 && a.N > 0 && a.K > 0, "vb_gemm: empty problem M=%d N=%d K=%d", a.M, a.N, a.K);
    VB_REQUIRE(a.N % 16 == 0, "vb_gemm: N=%d must be a multiple of 16", a.N);
    VB_REQUIRE(a.A && a.B && a.D, "vb_gemm: null operand");
    VB_REQUIRE(a.ldd % 16 == 0 && (reinterpret_cast<uintptr_t>(a.D) & 31) == 0, "vb_gemm: D must be 32-byte aligned with ldd a multiple of 16");
    VB_REQUIRE(!a.addend || (a.ld_add % 16 == 0 && (reinterpret_cast<uintptr_t>(a.addend) & 31) == 0), "vb_gemm: addend must be 32-byte aligned with ld a multiple of 16");
    VB_REQUIRE((!a.aux_in && !a.aux_out) || a.ld_aux % 16 == 0, "vb_gemm: ld_aux must be a multiple of 16");
    VB_REQUIRE((reinterpret_cast<uintptr_t>(a.aux_in) & 31) == 0 && (reinterpret_cast<uintptr_t>(a.aux_out) & 31) == 0,
               "vb_gemm: aux_in / aux_out must be 32-byte aligned");
    VB_REQUIRE(a.epilogue == VB_EPI_NONE || a.epilogue == VB_EPI_GELU || a.epilogue == VB_EPI_DGELU || a.epilogue == VB_EPI_GELU_FWD,
               "vb_gemm: unknown epilogue %d", a.epilogue);
    VB_REQUIRE(a.epilogue != VB_EPI_GELU || a.aux_out, "vb_gemm: GELU epilogue needs aux_out");
    VB_REQUIRE(a.epilogue != VB_EPI_DGELU || a.aux_in, "vb_gemm: DGELU epilogue needs aux_in");
    VB_REQUIRE(a.epilogue == VB_EPI_NONE || (!a.addend && a.dropout_p == 0.0f),
               "vb_gemm: the GELU / DGELU / GELU_FWD epilogues take no dropout and no addend");
    VB_REQUIRE(a.epilogue != VB_EPI_GELU_FWD || (!a.a_mn_major && !a.b_mn_major && !a.d_fp32 && !a.aux_in && !a.aux_out),
               "vb_gemm: the GELU_FWD epilogue needs K-major A and B and a bf16 D, and takes no aux_in / aux_out");
    VB_REQUIRE(!a.d_fp32 || (a.epilogue == VB_EPI_NONE && !a.addend && a.dropout_p == 0.0f),
               "vb_gemm: fp32-accumulate output supports bias only");
    VB_REQUIRE(a.dropout_p >= 0.0f && a.dropout_p < 1.0f, "vb_gemm: dropout_p out of range");
    VB_REQUIRE(!a.delta_out || (gemm_delta_ok(a.M, a.N) && a.delta_ctx && a.delta_seq > 0 && a.M % a.delta_seq == 0 && !a.d_fp32 &&
                                !a.a_mn_major && a.b_mn_major && !a.bias && !a.addend && a.dropout_p == 0.0f && a.epilogue == VB_EPI_NONE),
               "vb_gemm: delta_out needs a plain bf16 input-gradient GEMM (b_mn_major, no bias / addend / dropout) and vb_gemm_delta_ok(M, N)");
    // delta_ctx is read like an addend of row stride N (vb_gemm_delta_ok: N % 64 == 0), through a TMA tensor map
    VB_REQUIRE(!a.delta_out || (reinterpret_cast<uintptr_t>(a.delta_ctx) & 31) == 0, "vb_gemm: delta_ctx must be 32-byte aligned");
    VB_REQUIRE(!a.gp_tiled || (gemm_gp_tiled_ok(a.M, a.N) && !a.d_fp32 && !a.a_mn_major && (a.epilogue == VB_EPI_GELU || a.epilogue == VB_EPI_DGELU)),
               "vb_gemm: gp_tiled needs a GELU / DGELU epilogue and vb_gemm_gp_tiled_ok(M, N)");
    VB_REQUIRE(!a.gp_tiled || a.epilogue != VB_EPI_DGELU || a.b_mn_major,
               "vb_gemm: gp_tiled with the DGELU epilogue needs an MN-major B (the input-gradient GEMM)");
    VB_REQUIRE(!a.gp_tiled || a.epilogue != VB_EPI_GELU || !a.b_mn_major, "vb_gemm: gp_tiled with the GELU epilogue needs a K-major B");

    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = a.M; p.N = a.N; p.K = a.K;
    p.D = a.D; p.ldd = a.ldd;
    p.bias = a.bias;
    p.addend = static_cast<const bf16*>(a.addend); p.ld_add = a.ld_add;
    p.epilogue = a.epilogue;
    p.aux_in = static_cast<const bf16*>(a.aux_in);
    p.aux_out = static_cast<bf16*>(a.aux_out);
    p.ld_aux = a.ld_aux;
    if (a.delta_out) {   // O rides the residual-operand path of the epilogue (read, not added)
        p.addend = static_cast<const bf16*>(a.delta_ctx); p.ld_add = a.N;
        p.delta_out = a.delta_out; p.delta_seq = a.delta_seq;
    }
    p.m_fast = (a.M + BLOCK_M - 1) / BLOCK_M < (a.N + 255) / 256 ? 1 : 0;
    // the device seed offset of a dropout call (p.drop_offset shares its storage with delta_out: dispatch on this, not on p)
    const unsigned long long* const off = a.dropout_p > 0.0f ? drop_offset() : nullptr;
    if (a.dropout_p > 0.0f) {
        const DropQ q = dropout_quantise(a.dropout_p);
        p.drop_scale = q.scale;
        p.drop_thresh16 = q.thr8;
        p.drop_seed = a.dropout_seed;
        p.drop_stream = a.dropout_stream;
        if (off != nullptr) p.drop_offset = off;
    }

    const bool bn256 = use_bn256(a.N);
    VB_REQUIRE(!a.delta_out || bn256, "vb_gemm: delta_out needs 256-wide tiles");
    p.splits = a.d_fp32 ? wgrad_splits(gemm_tiles(a.M, a.N), gemm_k_blocks(a.K)) : 1;
    // Deterministic mode: the splits of an fp32 output store to their own slabs instead of red.add-ing one tile (one split is
    // already one writer per element). Slab kernels exist for the weight-gradient layout (A and B MN-major); other layouts,
    // and shapes whose slabs do not fit the workspace, lower the split factor to what fits, down to 1.
    const DetWs det = det_ws();
    if (a.d_fp32 && p.splits > 1 && det.ptr != nullptr) {
        const long long plane = static_cast<long long>(a.M) * a.N * 4;
        if (!(a.a_mn_major && a.b_mn_major)) p.splits = 1;
        while (p.splits > 1 && p.splits * plane > det.bytes) --p.splits;
    }
    const bool slab = a.d_fp32 && p.splits > 1 && det.ptr != nullptr;

    GemmMaps mp;
    memset(&mp, 0, sizeof(mp));
    if (!a.a_mn_major) VB_TRY_RC(make_tmap_bf16(&mp.a, a.A, a.K, a.M, a.lda, BLOCK_M));
    else               VB_TRY_RC(make_tmap_bf16(&mp.a, a.A, a.M, a.K, a.lda, BLOCK_K));
    if (!a.b_mn_major) VB_TRY_RC(make_tmap_bf16(&mp.b, a.B, a.K, a.N, a.ldb, bn256 ? 256 : 128));
    else               VB_TRY_RC(make_tmap_bf16(&mp.b, a.B, a.N, a.K, a.ldb, BLOCK_K));
    if (!a.d_fp32) {
        // bf16 outputs leave through TMA and the epilogue operand arrives through it: the argument checks above guarantee the
        // 16-byte alignment of every base and row stride that TMA needs (the tile-native gelu'(u) moves as contiguous bulk copies)
        if (!a.gp_tiled || a.epilogue != VB_EPI_GELU) VB_TRY_RC(make_tmap_bf16(&mp.d, a.D, a.N, a.M, a.ldd, 64));
        if (a.aux_out) VB_TRY_RC(make_tmap_bf16(&mp.x, a.aux_out, a.N, a.M, a.ld_aux, 64));
        if (p.addend) VB_TRY_RC(make_tmap_bf16(&mp.e, p.addend, a.N, a.M, p.ld_add, BLOCK_M));
        else if (a.aux_in && !a.gp_tiled) VB_TRY_RC(make_tmap_bf16(&mp.e, a.aux_in, a.N, a.M, a.ld_aux, BLOCK_M));
    }

    if (slab) {
        GemmParams q = p;
        q.D = det.ptr; q.ldd = a.N; q.bias = nullptr;
        const int rc2 = bn256 ? launch<true, true, 256, true, EPI_SLAB>(mp, q, st) : launch<true, true, 128, true, EPI_SLAB>(mp, q, st);
        if (rc2) return rc2;
        const long long n4 = static_cast<long long>(a.M) * a.N / 4;
        long long blocks = (n4 + 255) / 256;
        if (blocks > num_sms() * 8) blocks = num_sms() * 8;
        {
            ProfScope ps(st, PROF_GEMM_WGRAD, 0.0, 1);
            splitk_reduce_kernel<<<static_cast<int>(blocks), 256, 0, st>>>(static_cast<const float*>(det.ptr), p.splits, a.M, a.N, a.bias,
                                                                           static_cast<float*>(a.D), a.ldd);
        }
        VB_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    if (off != nullptr) {
        // dropout with the seed offset in device memory: the generic epilogue (it applies bias, dropout and addend in the order of
        // the specialised ones, so the bits equal a call with seed + *offset by value)
#define VB_DISPATCH_OFF(AM, BM) \
    (bn256 ? launch<AM, BM, 256, false, EPI_GENERIC_OFF>(mp, p, st) : launch<AM, BM, 128, false, EPI_GENERIC_OFF>(mp, p, st))
        if (!a.a_mn_major && !a.b_mn_major) return VB_DISPATCH_OFF(false, false);
        if (!a.a_mn_major && a.b_mn_major) return VB_DISPATCH_OFF(false, true);
        if (a.a_mn_major && a.b_mn_major) return VB_DISPATCH_OFF(true, true);
        return VB_DISPATCH_OFF(true, false);
#undef VB_DISPATCH_OFF
    }
    if (a.epilogue == VB_EPI_GELU_FWD)
        return bn256 ? launch<false, false, 256, false, EPI_GELU_ONLY>(mp, p, st) : launch<false, false, 128, false, EPI_GELU_ONLY>(mp, p, st);
    if (bn256 && !a.d_fp32) {
        // specialised epilogues for the shapes of the layer (forward and input-gradient GEMMs); anything else: generic
        const bool drop = a.dropout_p > 0.0f, add = a.addend != nullptr;
        int epi = EPI_GENERIC;
        if (a.epilogue == VB_EPI_GELU) epi = a.gp_tiled ? EPI_GELU_FWD_T : EPI_GELU_FWD;
        else if (a.epilogue == VB_EPI_DGELU) epi = a.gp_tiled ? EPI_DGELU_BWD_T : EPI_DGELU_BWD;
        else epi = add ? (drop ? EPI_DROP_RESID : EPI_RESID) : (drop ? EPI_GENERIC : EPI_BIAS);
        if (a.delta_out) epi = EPI_DELTA;
        if (!a.a_mn_major && !a.b_mn_major) {
            switch (epi) {
                case EPI_BIAS: return launch<false, false, 256, false, EPI_BIAS>(mp, p, st);
                case EPI_RESID: return launch<false, false, 256, false, EPI_RESID>(mp, p, st);
                case EPI_DROP_RESID: return launch<false, false, 256, false, EPI_DROP_RESID>(mp, p, st);
                case EPI_GELU_FWD: return launch<false, false, 256, false, EPI_GELU_FWD>(mp, p, st);
                case EPI_GELU_FWD_T: return launch<false, false, 256, false, EPI_GELU_FWD_T>(mp, p, st);
                default: return launch<false, false, 256, false>(mp, p, st);
            }
        }
        if (!a.a_mn_major && a.b_mn_major) {
            switch (epi) {
                case EPI_BIAS: return launch<false, true, 256, false, EPI_BIAS>(mp, p, st);
                case EPI_RESID: return launch<false, true, 256, false, EPI_RESID>(mp, p, st);
                case EPI_DGELU_BWD: return launch<false, true, 256, false, EPI_DGELU_BWD>(mp, p, st);
                case EPI_DELTA: return launch<false, true, 256, false, EPI_DELTA>(mp, p, st);
                case EPI_DGELU_BWD_T: return launch<false, true, 256, false, EPI_DGELU_BWD_T>(mp, p, st);
                default: return launch<false, true, 256, false>(mp, p, st);
            }
        }
    }

#define VB_DISPATCH(AM, BM, F32)                                         \
    (bn256 ? launch<AM, BM, 256, F32>(mp, p, st) : launch<AM, BM, 128, F32>(mp, p, st))
    if (!a.d_fp32) {
        if (!a.a_mn_major && !a.b_mn_major) return VB_DISPATCH(false, false, false);
        if (!a.a_mn_major && a.b_mn_major) return VB_DISPATCH(false, true, false);
        if (a.a_mn_major && a.b_mn_major) return VB_DISPATCH(true, true, false);
        return VB_DISPATCH(true, false, false);
    } else {
        if (!a.a_mn_major && !a.b_mn_major) return VB_DISPATCH(false, false, true);
        if (!a.a_mn_major && a.b_mn_major) return VB_DISPATCH(false, true, true);
        if (a.a_mn_major && a.b_mn_major) return VB_DISPATCH(true, true, true);
        return VB_DISPATCH(true, false, true);
    }
#undef VB_DISPATCH
}

}  // namespace vb

extern "C" {
int vb_abi_version(void) { return VB_ABI_VERSION; }
const char* vb_last_error(void) { return vb::get_error(); }
int64_t vb_launch_count(void) { return vb::g_launches.load(); }
void vb_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(vb::g_prof_mu);
    vb::g_prof_on = on != 0;
}
int vb_profile_read(double* ms, double* work, int64_t* launches) {
    if (cudaDeviceSynchronize() != cudaSuccess) { vb::set_error("vb_profile_read: device sync failed"); return 1; }
    std::lock_guard<std::mutex> lk(vb::g_prof_mu);
    for (int c = 0; c < vb::PROF_NCAT; ++c) { ms[c] = 0; work[c] = 0; launches[c] = 0; }
    for (auto& r : vb::g_prof) {
        float t = 0.f;
        cudaEventElapsedTime(&t, r.e0, r.e1);
        ms[r.cat] += t; work[r.cat] += r.work; launches[r.cat] += r.launches;
        vb::g_prof_pool.push_back(r);
    }
    vb::g_prof.clear();
    return 0;
}
int vb_set_deterministic(void* workspace, int64_t bytes) {
    if (workspace != nullptr && (bytes <= 0 || (reinterpret_cast<uintptr_t>(workspace) & 255) != 0)) {
        vb::set_error("vb_set_deterministic: the workspace must be 256-byte aligned and bytes > 0 (got %p, %lld)", workspace,
                      static_cast<long long>(bytes));
        return 2;
    }
    vb::g_det_ptr = workspace;
    vb::g_det_bytes = workspace != nullptr ? bytes : 0;
    return 0;
}
int vb_set_dropout_offset(const uint64_t* offset) {
    if ((reinterpret_cast<uintptr_t>(offset) & 7) != 0) {
        vb::set_error("vb_set_dropout_offset: the offset must be 8-byte aligned (got %p)", static_cast<const void*>(offset));
        return 2;
    }
    vb::g_drop_offset = reinterpret_cast<const unsigned long long*>(offset);
    return 0;
}
int vb_gemm_delta_ok(int32_t M, int32_t N) { return vb::gemm_delta_ok(M, N) ? 1 : 0; }
int vb_gemm_gp_tiled_ok(int32_t M, int32_t N) { return vb::gemm_gp_tiled_ok(M, N) ? 1 : 0; }
int vb_gemm(const vb_gemm_args* args, void* stream) {
    if (!args) { vb::set_error("vb_gemm: null args"); return 2; }
    return vb::gemm(*args, static_cast<cudaStream_t>(stream));
}
}
