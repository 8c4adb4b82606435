// vb_gemm.cu — the dense-contraction core of the VisualBERT encoder hot path on sm_90a.
//
// One warp-specialised kernel computes D[M,N] = epi(sum_k A(m,k) B(n,k)) in bf16 with fp32 accumulation,
// one 128 x BLOCK_N tile per CTA (BLOCK_N = 256, or 128 for narrow / ragged N):
//   warpgroup 0     TMA producer  (one elected thread: cp.async.bulk.tensor, 128B-swizzled 64-wide k-slabs,
//                                  4-stage mbarrier ring)
//   warpgroups 1-2  MMA + epilogue (wgmma.mma_async 64 x 128 x 16 from shared-memory descriptors, fp32 accumulators in
//                                  registers, 64 rows per warpgroup; then the tile goes through shared memory so that a
//                                  thread owns 16-column pieces of one row for bias / dropout / residual / GELU / GELU'
//                                  and 32-byte stores, or fp32 red.add for split-K weight gradients)
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
    // fp32 accumulator tile for the epilogue, written over the drained operand ring; +4 floats per row keeps the
    // row-per-lane reads of the epilogue free of bank conflicts
    static constexpr int ACC_LD = BLOCK_N + 4;
    static constexpr int RING_BYTES = kStages * STAGE_BYTES > BLOCK_M * ACC_LD * 4 ? kStages * STAGE_BYTES : BLOCK_M * ACC_LD * 4;
    static constexpr int BAR_OFF = RING_BYTES;
    static constexpr int NUM_BARS = 2 * kStages;
    static constexpr int BIAS_OFF = BAR_OFF + NUM_BARS * 8;
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

// Epilogue for 16 consecutive columns of one row held as fp32 in x[16]. All global traffic is
// 32 bytes per thread per access (two 128-bit accesses): a thread owns a row, so 32-byte pieces are the
// unit that keeps every DRAM/L2 sector fully written.
__device__ __forceinline__ void load16_bf16(const bf16* p, float (&f)[16]) {
    uint32_t r[8];
    ldg_v8(p, r);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float2 t = unpack_bf16x2(r[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}
__device__ __forceinline__ void store16_bf16(bf16* p, const float (&f)[16]) {
    uint32_t r[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) r[i] = pack_bf16x2(f[2 * i], f[2 * i + 1]);
    stg_v8(p, r);
}

// `sbias` points at the 16 staged bias values of these columns in shared memory (or nullptr).
// `ex` holds the 16 bf16 of the residual (addend) or of gelu'(u) (aux_in) for these columns, prefetched by the
// caller before the accumulators are staged, so the row-strided global load never sits on the critical path.
// EPI selects the epilogue at COMPILE time: the generic form (every option a run-time branch, all chunks unrolled) is several
// times larger than one specialised path, and instruction-cache misses then stall the epilogue. A specialised kernel carries
// only its path.
// _T: gelu'(u) is kept in the TILE-NATIVE layout (vb_gemm_args.gp_tiled): the only reader of that tensor is the epilogue of the
// backward GEMM, where the same thread holds the same 16 columns — so it is stored in 1 KB blocks (one per epilogue warp and
// chunk, row r of the warp's 32 at block + 32 r bytes) that both epilogues access in contiguous pieces.
// EPI_DELTA: plain bf16 store plus the attention backward's D[b, head, s] = sum_d dO[row, head, d] * O[row, head, d] (vb_gemm_args.delta_*):
// the GEMM that PRODUCES dO (input gradient of attention.output.dense) has, in each epilogue thread, 128 consecutive columns of one row —
// two whole heads — so the row-wise dot product with O needs no exchange; O is read like a residual operand.
// EPI_GELU_ONLY (VB_EPI_GELU_FWD of the ABI): D = gelu(u) and nothing else — the forward-only FFN-up GEMM. It takes the plain
// bf16 store path (one coalesced store per element) with the gelu of the two-tensor epilogues.
// EPI_SLAB (fp32 output, deterministic mode): split s STORES its partial tile to slab s of the workspace, D = slab base with
// ldd = N, slab s at D + s * M * N, no bias; splitk_reduce_kernel then adds bias + the slabs in split order into the real D.
enum { EPI_GENERIC = 0, EPI_BIAS = 1, EPI_RESID = 2, EPI_DROP_RESID = 3, EPI_GELU_FWD = 4, EPI_DGELU_BWD = 5, EPI_GELU_FWD_T = 6,
       EPI_DGELU_BWD_T = 7, EPI_DELTA = 8, EPI_GELU_ONLY = 9, EPI_SLAB = 10, EPI_GENERIC_OFF = 11 };
// EPI_GENERIC_OFF: the generic epilogue with the dropout seed p.drop_seed + *p.drop_offset, read from device memory when the
// epilogue runs (vb_set_dropout_offset); a call with dropout takes it whenever an offset is set, so no other kernel reads it.
__host__ __device__ constexpr bool epi_is_generic(int e) { return e == EPI_GENERIC || e == EPI_GENERIC_OFF; }
__host__ __device__ constexpr bool epi_is_gelu(int e) { return e == EPI_GELU_FWD || e == EPI_GELU_FWD_T; }
__host__ __device__ constexpr bool epi_is_dgelu(int e) { return e == EPI_DGELU_BWD || e == EPI_DGELU_BWD_T; }

// TO_REGS: nothing is stored; the 16 bf16 results are returned packed in o0 (what goes to D) and, for the GELU epilogue,
// o1 (what goes to aux_out) — the caller stores them.
template <bool OUT_F32, int EPI = EPI_GENERIC, bool TO_REGS = false>
__device__ __forceinline__ void epilogue16(const GemmParams& p, int row, int col, const float* sbias, const uint32_t (&ex)[8],
                                           float (&x)[16], uint32_t* o0 = nullptr, uint32_t* o1 = nullptr) {
    if (sbias != nullptr) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float4 b = *reinterpret_cast<const float4*>(sbias + 4 * i);  // warp-uniform address: broadcast
            x[4 * i] += b.x; x[4 * i + 1] += b.y; x[4 * i + 2] += b.z; x[4 * i + 3] += b.w;
        }
    }
    if constexpr (OUT_F32) {
        float* d = reinterpret_cast<float*>(p.D) + static_cast<long long>(row) * p.ldd + col;
#pragma unroll
        for (int i = 0; i < 4; ++i) red_add_v4_f32(d + 4 * i, x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
    } else {
        constexpr bool kGeneric = epi_is_generic(EPI);
        if (EPI == EPI_DROP_RESID || (kGeneric && p.drop_scale != 0.0f)) {
            const unsigned long long e8 =
                (static_cast<unsigned long long>(row) * static_cast<unsigned>(p.N) + col) >> 3;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t keep = dropout_keep8(EPI == EPI_GENERIC_OFF ? p.drop_seed + *p.drop_offset : p.drop_seed, p.drop_stream, e8 + h,
                                                    p.drop_thresh16);
#pragma unroll
                for (int i = 0; i < 8; ++i) x[8 * h + i] = ((keep >> i) & 1u) ? x[8 * h + i] * p.drop_scale : 0.0f;
            }
        }
        if (EPI == EPI_RESID || EPI == EPI_DROP_RESID || (kGeneric && p.addend != nullptr)) {   // (EPI_DELTA reads ex in the caller)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float2 t = unpack_bf16x2(ex[i]);
                x[2 * i] += t.x;
                x[2 * i + 1] += t.y;
            }
        }
        bf16* d = reinterpret_cast<bf16*>(p.D) + static_cast<long long>(row) * p.ldd + col;
        if (EPI == EPI_GELU_ONLY) {
            // D <- gelu(u): the value the GELU epilogue below sends to aux_out, from the same function; its derivative is dropped
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                float gp;
                gelu_fwd_bwd(x[i], x[i], gp);
            }
        } else if (epi_is_gelu(EPI) || (kGeneric && p.epilogue == VB_EPI_GELU)) {
            // aux_out <- gelu(u) (operand of the next GEMM), D <- gelu'(u) (all the backward needs of u)
            float gp[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) gelu_fwd_bwd(x[i], x[i], gp[i]);
            if constexpr (TO_REGS) {
#pragma unroll
                for (int i = 0; i < 8; ++i) { o0[i] = pack_bf16x2(gp[2 * i], gp[2 * i + 1]); o1[i] = pack_bf16x2(x[2 * i], x[2 * i + 1]); }
                return;
            }
            store16_bf16(d, gp);
            d = p.aux_out + static_cast<long long>(row) * p.ld_aux + col;
        } else if (epi_is_dgelu(EPI) || (kGeneric && p.epilogue == VB_EPI_DGELU)) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float2 t = unpack_bf16x2(ex[i]);
                x[2 * i] *= t.x;
                x[2 * i + 1] *= t.y;
            }
        }
        if constexpr (TO_REGS) {
#pragma unroll
            for (int i = 0; i < 8; ++i) o0[i] = pack_bf16x2(x[2 * i], x[2 * i + 1]);
            return;
        }
        store16_bf16(d, x);
    }
}

template <bool A_MN, bool B_MN, int BLOCK_N, bool OUT_F32, int EPI = EPI_GENERIC>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
    using C = Cfg<BLOCK_N>;
    static_assert(BLOCK_N % 128 == 0, "64 x 128 wgmma pieces");
    static_assert(!(EPI == EPI_GELU_FWD_T || EPI == EPI_DGELU_BWD_T) || BLOCK_N == 256, "tile-native gelu' is defined on 256-wide tiles");
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

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 2);   // one arrival per MMA warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();  // everything above is on-chip set-up; operands of the previous kernel are read only from here on

    const int m_blocks = (p.M + BLOCK_M - 1) / BLOCK_M;
    const int n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
    const int k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
    const TileCoord tc = decode_tile(blockIdx.x, n_blocks, p.splits, k_blocks, m_blocks, p.m_fast != 0);

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
    constexpr int NH = BLOCK_N / 128;
    // K-major: advance 16 elements (32 B) inside the swizzle row; MN-major: 16 k-rows (2 KB)
    constexpr uint32_t a_kstep = A_MN ? WGMMA_K * 128 : WGMMA_K * 2;
    constexpr uint32_t b_kstep = B_MN ? WGMMA_K * 128 : WGMMA_K * 2;
    float acc[NH][64];
    {
        int stage = 0, prev = 0;
        uint32_t phase = 0;
        for (int kb = tc.kb_begin; kb < tc.kb_end; ++kb) {
            mbar_wait(full_bar(stage), phase);
            // this warpgroup's 64 rows of A: 64 K-major rows or one 64-wide MN-major atom = 8 KB further in both layouts;
            // the second 128 columns of B likewise start 16 KB further
            const uint32_t a0 = a_tile(stage) + wg * 8192, b0 = b_tile(stage);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
                const uint64_t ad = wgmma_desc_sw128(a0 + k * a_kstep, kAtomBytes, 1024);
#pragma unroll
                for (int h = 0; h < NH; ++h)
                    wgmma_m64n128k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[h], ad, wgmma_desc_sw128(b0 + h * 16384 + k * b_kstep, kAtomBytes, 1024),
                                                                 (kb > tc.kb_begin || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
            // the MMAs of the previous k-block have retired: its slot may be refilled
            wgmma_wait<1>();
            if (kb > tc.kb_begin && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar(prev));
            prev = stage;
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
    }

    // ---------------- epilogue ----------------
    // Thread -> element map: epilogue warp ew owns rows 32 (ew % 4) .. + 31 and the column half ew / 4 of the tile, in 16-column
    // chunks; in step j a thread holds one chunk of one row. By default lane l takes chunk l / RPI of row RPI j + l % RPI of the
    // warp's 32, so that one warp access covers RPI whole half-rows (RPI x 256 contiguous bytes of a bf16 output instead of 32
    // bytes of 32 rows), and the staging reads of a quarter-warp hit 8 distinct 4-bank groups (ACC_LD = 4 mod 32). EPI_DELTA keeps
    // one row per lane and chunk j in step j: a thread then holds whole heads of its row.
    // Operands read by the epilogue (residual / gelu') are requested before the accumulators are staged.
    const int ew = warp - 4;
    const int q = ew & 3, half = ew >> 2;
    const int col0 = tc.n_blk * BLOCK_N + half * (BLOCK_N / 2);
    constexpr int NCH = BLOCK_N / 2 / 16;
    constexpr int RPI = 32 / NCH;
    constexpr bool kRowPerLane = EPI == EPI_DELTA;
    auto wrow_of = [&](int j) { return kRowPerLane ? lane : RPI * j + lane % RPI; };   // row within the warp's 32
    auto chunk_of = [&](int j) { return kRowPerLane ? j : lane / RPI; };
    // tile-native gelu'(u) (M, N multiples of 256; vbert_b200.h): 1 KB warp blocks per chunk, row r of the warp's 32 at + 32 r bytes
    const long long gp_warp_off =
        ((((static_cast<long long>(tc.m_blk >> 1) * n_blocks + tc.n_blk) * 2 + (tc.m_blk & 1)) * kEpiWarps + ew) * NCH) * 512;
    auto gp_off = [&](int j) { return gp_warp_off + chunk_of(j) * 512 + wrow_of(j) * 16; };
    constexpr bool kEx = !OUT_F32 && EPI != EPI_BIAS && !epi_is_gelu(EPI) && EPI != EPI_GELU_ONLY;
    uint32_t ex[kEx ? NCH : 1][8];
    if constexpr (kEx) {
        constexpr bool kWantAdd = EPI == EPI_RESID || EPI == EPI_DROP_RESID || EPI == EPI_DELTA;   // EPI_DELTA: addend = O
        const int row0 = tc.m_blk * BLOCK_M + q * 32 + wrow_of(0), c0 = col0 + chunk_of(0) * 16;   // step j: row0 + (row step) j
        const bf16* exb = nullptr;
        long long ex_step = 0;
        if (kWantAdd || (epi_is_generic(EPI) && p.addend != nullptr)) {
            exb = p.addend + static_cast<long long>(row0) * p.ld_add + c0;
            ex_step = kRowPerLane ? 16 : RPI * p.ld_add;
        } else if (EPI == EPI_DGELU_BWD || (epi_is_generic(EPI) && p.epilogue == VB_EPI_DGELU)) {
            exb = p.aux_in + static_cast<long long>(row0) * p.ld_aux + c0;
            ex_step = kRowPerLane ? 16 : RPI * p.ld_aux;
        } else if (EPI == EPI_DGELU_BWD_T) {
            exb = p.aux_in + gp_off(0);
            ex_step = kRowPerLane ? 512 : RPI * 16;
        }
#pragma unroll
        for (int j = 0; j < NCH; ++j)
            if (exb != nullptr && tc.m_blk * BLOCK_M + q * 32 + wrow_of(j) < p.M && col0 + chunk_of(j) * 16 < p.N) ldg_v8(exb + j * ex_step, ex[j]);
    }

    // both warpgroups' MMAs have retired (and with them every read of the ring): stage the accumulators over the ring
    named_bar_sync(1, kEpiWarps * 32);
    float* sacc = reinterpret_cast<float*>(smem);
    {
        const int r0 = wg * 64 + ((warp & 3) << 4) + (lane >> 2);
#pragma unroll
        for (int h = 0; h < NH; ++h)
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i)
                    *reinterpret_cast<float2*>(sacc + (r0 + 8 * i) * C::ACC_LD + h * 128 + j * 8 + 2 * (lane & 3)) =
                        make_float2(acc[h][4 * j + 2 * i], acc[h][4 * j + 2 * i + 1]);
    }
    named_bar_sync(1, kEpiWarps * 32);

    [[maybe_unused]] float hsum = 0.f;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
        const int lrow = q * 32 + wrow_of(k), cc = half * (BLOCK_N / 2) + chunk_of(k) * 16;   // in the tile
        const int row = tc.m_blk * BLOCK_M + lrow;
        const int col = tc.n_blk * BLOCK_N + cc;
        if (row < p.M && col < p.N) {
            float x[16];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 v = *reinterpret_cast<const float4*>(sacc + lrow * C::ACC_LD + cc + 4 * i);
                x[4 * i] = v.x; x[4 * i + 1] = v.y; x[4 * i + 2] = v.z; x[4 * i + 3] = v.w;
            }
            const float* sb = has_bias ? sbias + cc : nullptr;
            const uint32_t (&e)[8] = ex[kEx ? k : 0];
            if constexpr (EPI == EPI_GELU_FWD_T) {
                // gelu'(u) into the tile-native buffer, gelu(u) row-major
                uint32_t o0[8], o1[8];
                epilogue16<OUT_F32, EPI, true>(p, row, col, sb, e, x, o0, o1);
                stg_v8(reinterpret_cast<bf16*>(p.D) + gp_off(k), o0);
                stg_v8(p.aux_out + static_cast<long long>(row) * p.ld_aux + col, o1);
            } else if constexpr (EPI == EPI_SLAB) {
                float* d = reinterpret_cast<float*>(p.D) + (static_cast<long long>(blockIdx.x / (m_blocks * n_blocks)) * p.M + row) * p.ldd + col;
#pragma unroll
                for (int i = 0; i < 4; ++i) *reinterpret_cast<float4*>(d + 4 * i) = make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
            } else if constexpr (EPI == EPI_DELTA) {
                uint32_t o0[8];
                epilogue16<OUT_F32, EPI, true>(p, row, col, sb, e, x, o0);
                stg_v8(reinterpret_cast<bf16*>(p.D) + static_cast<long long>(row) * p.ldd + col, o0);
#pragma unroll
                for (int i = 0; i < 8; ++i) {   // dot product of the ROUNDED dO (what the attention kernel will read) with O
                    const float2 a = unpack_bf16x2(o0[i]), b = unpack_bf16x2(e[i]);
                    hsum = fmaf(a.x, b.x, fmaf(a.y, b.y, hsum));
                }
            } else {
                epilogue16<OUT_F32, EPI>(p, row, col, sb, e, x);
            }
        }
        if constexpr (EPI == EPI_DELTA) {
            if ((k & 3) == 3) {   // four chunks are exactly one head (col0 is a multiple of 64)
                const int c4 = col - 48;
                if (row < p.M && c4 < p.N) {
                    const int bi = row / p.delta_seq, si = row - bi * p.delta_seq;
                    p.delta_out[(static_cast<long long>(bi) * (p.N >> 6) + (c4 >> 6)) * p.delta_seq + si] = hsum;
                }
                hsum = 0.f;
            }
        }
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

template <bool A_MN, bool B_MN, int BLOCK_N, bool OUT_F32, int EPI = EPI_GENERIC>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t st) {
    using C = Cfg<BLOCK_N>;
    auto kern = gemm_wgmma_kernel<A_MN, B_MN, BLOCK_N, OUT_F32, EPI>;
    static int configured[kMaxDevices] = {0};
    VB_CHECK_CUDA(ensure_dyn_smem(kern, C::SMEM_BYTES, configured));
    const long long tiles = static_cast<long long>((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N) * p.splits;
    VB_REQUIRE(tiles < (1LL << 31), "vb_gemm: too many tiles");
    {
        ProfScope ps(st, OUT_F32 ? PROF_GEMM_WGRAD : (B_MN ? PROF_GEMM_DGRAD : PROF_GEMM_FWD), 2.0 * p.M * p.N * p.K, 1);
        VB_CHECK_CUDA(launch_pdl(kern, dim3(static_cast<unsigned>(tiles)), dim3(kThreads), C::SMEM_BYTES, st, ta, tb, p));
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
                                !a.a_mn_major && a.b_mn_major && !a.bias && !a.addend && a.dropout_p == 0.0f && a.epilogue == VB_EPI_NONE &&
                                (reinterpret_cast<uintptr_t>(a.delta_ctx) & 31) == 0),
               "vb_gemm: delta_out needs a plain bf16 input-gradient GEMM (b_mn_major, no bias / addend / dropout) and vb_gemm_delta_ok(M, N)");
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

    CUtensorMap ta, tb;
    int rc;
    if (!a.a_mn_major) rc = make_tmap_bf16(&ta, a.A, a.K, a.M, a.lda, BLOCK_M);
    else               rc = make_tmap_bf16(&ta, a.A, a.M, a.K, a.lda, BLOCK_K);
    if (rc) return rc;
    if (!a.b_mn_major) rc = make_tmap_bf16(&tb, a.B, a.K, a.N, a.ldb, bn256 ? 256 : 128);
    else               rc = make_tmap_bf16(&tb, a.B, a.N, a.K, a.ldb, BLOCK_K);
    if (rc) return rc;

    if (slab) {
        GemmParams q = p;
        q.D = det.ptr; q.ldd = a.N; q.bias = nullptr;
        const int rc2 = bn256 ? launch<true, true, 256, true, EPI_SLAB>(ta, tb, q, st) : launch<true, true, 128, true, EPI_SLAB>(ta, tb, q, st);
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
    (bn256 ? launch<AM, BM, 256, false, EPI_GENERIC_OFF>(ta, tb, p, st) : launch<AM, BM, 128, false, EPI_GENERIC_OFF>(ta, tb, p, st))
        if (!a.a_mn_major && !a.b_mn_major) return VB_DISPATCH_OFF(false, false);
        if (!a.a_mn_major && a.b_mn_major) return VB_DISPATCH_OFF(false, true);
        if (a.a_mn_major && a.b_mn_major) return VB_DISPATCH_OFF(true, true);
        return VB_DISPATCH_OFF(true, false);
#undef VB_DISPATCH_OFF
    }
    if (a.epilogue == VB_EPI_GELU_FWD)
        return bn256 ? launch<false, false, 256, false, EPI_GELU_ONLY>(ta, tb, p, st) : launch<false, false, 128, false, EPI_GELU_ONLY>(ta, tb, p, st);
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
                case EPI_BIAS: return launch<false, false, 256, false, EPI_BIAS>(ta, tb, p, st);
                case EPI_RESID: return launch<false, false, 256, false, EPI_RESID>(ta, tb, p, st);
                case EPI_DROP_RESID: return launch<false, false, 256, false, EPI_DROP_RESID>(ta, tb, p, st);
                case EPI_GELU_FWD: return launch<false, false, 256, false, EPI_GELU_FWD>(ta, tb, p, st);
                case EPI_GELU_FWD_T: return launch<false, false, 256, false, EPI_GELU_FWD_T>(ta, tb, p, st);
                default: return launch<false, false, 256, false>(ta, tb, p, st);
            }
        }
        if (!a.a_mn_major && a.b_mn_major) {
            switch (epi) {
                case EPI_BIAS: return launch<false, true, 256, false, EPI_BIAS>(ta, tb, p, st);
                case EPI_RESID: return launch<false, true, 256, false, EPI_RESID>(ta, tb, p, st);
                case EPI_DGELU_BWD: return launch<false, true, 256, false, EPI_DGELU_BWD>(ta, tb, p, st);
                case EPI_DELTA: return launch<false, true, 256, false, EPI_DELTA>(ta, tb, p, st);
                case EPI_DGELU_BWD_T: return launch<false, true, 256, false, EPI_DGELU_BWD_T>(ta, tb, p, st);
                default: return launch<false, true, 256, false>(ta, tb, p, st);
            }
        }
    }

#define VB_DISPATCH(AM, BM, F32)                                         \
    (bn256 ? launch<AM, BM, 256, F32>(ta, tb, p, st) : launch<AM, BM, 128, F32>(ta, tb, p, st))
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
