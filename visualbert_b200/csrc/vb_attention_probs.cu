// vb_attention_probs.cu — the attention maps softmax(QK^T / 8 + mask) [B, A, S, S] in fp32, pre-dropout
// (reference M.py:241-247, returned by the output_attention_weights mode, M.py:258-259, 1316-1324).
//
// The fused attention kernels never write P; this kernel materialises it from the bf16 Q and K of the layer's qkv, the
// same operands and the same fp32 exp2-domain arithmetic as the forward kernels. One CTA = (64 query rows, head, batch),
// 4 warps x 16 rows, K streamed in 64-key tiles through a two-slot cp.async ring. Two passes over the keys: pass 1 keeps
// the row max and sum (online, per thread, then combined over the quad), pass 2 recomputes the scores and stores
// exp2(s - max) / sum. The statistics are the kernel's own rather than the forward's saved lse: in an example whose keys
// are all masked the lse is about -10000 and fp32 holds it to 2^-10, which would cost 5e-4 relative in every
// probability of that example. Here the mask is shifted by the example's largest key bias first (exact for the 0 /
// -10000 masks), so such rows come out as softmax(QK^T / 8) to fp32 rounding, as the reference defines them.
// The QK^T products are computed twice; at 2 x 128 FLOP per 4-byte output element the kernel stays bound by its stores.
//
// Stores: the m16n8 accumulator layout gives a thread 2 adjacent columns of 2 rows, i.e. 8-byte pieces of 8 rows per
// warp instruction. A warp stages its 16 x 64 fp32 tile in shared memory and writes it back row by row, lane l taking
// columns l and l + 32: every store instruction writes 128 contiguous bytes of one row, whatever the (possibly odd)
// row length S. Every element of [B, A, S, S] is written exactly once; masked keys give exact zeros (exp2 of about
// -14400 flushes to 0), rows and columns >= S are neither read nor written.
#include "vb_attention.cuh"
#include "vb_internal.h"

namespace vb {

constexpr int kProbsLd = kBlk + 4;  // staging row stride in floats: the float2 writes of a quad's 8 rows spread over the banks

__global__ void __launch_bounds__(128)
attn_probs_kernel(const bf16* __restrict__ qkv, const float* __restrict__ mask_bias, float* __restrict__ probs, int S, int A,
                  int H) {
    extern __shared__ __align__(128) uint8_t dsmem[];
    __shared__ float sred[4];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int nkb = (S + kBlk - 1) / kBlk;
    const uint32_t sQ = smem_u32(dsmem), sK0 = sQ + kTileBytes;  // Q | K ring [2]
    float* stage = reinterpret_cast<float*>(dsmem + 3 * kTileBytes) + warp * 16 * kProbsLd;
    float* sbias = reinterpret_cast<float*>(dsmem + 3 * kTileBytes) + 4 * 16 * kProbsLd;  // [nkb * 64], exp2 domain
    const long long ld = 3LL * H;
    const bf16* qbase = qkv + static_cast<long long>(b) * S * ld + h * kHd;
    const bf16* kbase = qbase + H;
    const int qrow0 = qb * kBlk + warp * 16;
    const bool active = qrow0 < S;
    pdl_trigger();
    pdl_wait();

    load_tile(sQ, qbase, ld, qb * kBlk, S, tid);
    load_tile(sK0, kbase, ld, 0, S, tid);
    cp_async_commit();
    // key bias relative to the example's largest one (mask_bias[b, j] - c is exact for biases within a factor 2 of c)
    const float* mb = mask_bias + static_cast<long long>(b) * S;
    float c = -INFINITY;
    for (int j = tid; j < S; j += 128) c = fmaxf(c, mb[j]);
    c = warp_max(c);
    if (lane == 0) sred[warp] = c;
    __syncthreads();
    c = fmaxf(fmaxf(sred[0], sred[1]), fmaxf(sred[2], sred[3]));
    for (int j = tid; j < nkb * kBlk; j += 128) sbias[j] = j < S ? (mb[j] - c) * kLog2e : -INFINITY;

    const float sc2 = 0.125f * kLog2e;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    uint32_t qf[4][4];
    const int steps = 2 * nkb;  // pass 1: key blocks 0 .. nkb-1, pass 2: the same again
    for (int step = 0; step < steps; ++step) {
        if (step + 1 < steps) {
            load_tile(sK0 + ((step + 1) & 1) * kTileBytes, kbase, ld, ((step + 1) % nkb) * kBlk, S, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();  // tile `step` (and at step 0 Q and sbias) visible to every warp
        if (active) {
            if (step == 0) load_afrag(qf, sQ, warp * 16, lane);
            const int kb = step % nkb;
            const int kvalid = min(kBlk, S - kb * kBlk);
            float s[8][4];
            zero_acc(s);
            gemm_nt(s, qf, sK0 + (step & 1) * kTileBytes, lane, kvalid);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const float b0 = sbias[kb * kBlk + nt * 8 + 2 * t], b1 = sbias[kb * kBlk + nt * 8 + 2 * t + 1];
                s[nt][0] = fmaf(s[nt][0], sc2, b0); s[nt][1] = fmaf(s[nt][1], sc2, b1);
                s[nt][2] = fmaf(s[nt][2], sc2, b0); s[nt][3] = fmaf(s[nt][3], sc2, b1);
            }
            if (step < nkb) {  // pass 1: this thread's running max / sum of rows g and g + 8
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    float mx = -INFINITY;
#pragma unroll
                    for (int nt = 0; nt < 8; ++nt) mx = fmaxf(mx, fmaxf(s[nt][2 * r], s[nt][2 * r + 1]));
                    const float mn = fmaxf(m[r], mx);
                    if (mn != -INFINITY) {  // keys >= S are -inf: a thread may not have seen a valid key yet
                        float sum = 0.f;
#pragma unroll
                        for (int nt = 0; nt < 8; ++nt) sum += fast_ex2(s[nt][2 * r] - mn) + fast_ex2(s[nt][2 * r + 1] - mn);
                        l[r] = l[r] * fast_ex2(m[r] - mn) + sum;
                        m[r] = mn;
                    }
                }
                if (step == nkb - 1) {  // combine the quad's partial statistics of each row
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        float mq = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
                        mq = fmaxf(mq, __shfl_xor_sync(0xffffffffu, mq, 2));
                        float lq = m[r] == -INFINITY ? 0.f : l[r] * fast_ex2(m[r] - mq);
                        lq += __shfl_xor_sync(0xffffffffu, lq, 1);
                        lq += __shfl_xor_sync(0xffffffffu, lq, 2);
                        m[r] = mq;
                        l[r] = 1.f / lq;
                    }
                }
            } else {  // pass 2: probabilities -> staging tile -> 128-byte row segments
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const int col = nt * 8 + 2 * t;
                    *reinterpret_cast<float2*>(stage + g * kProbsLd + col) =
                        make_float2(fast_ex2(s[nt][0] - m[0]) * l[0], fast_ex2(s[nt][1] - m[0]) * l[0]);
                    *reinterpret_cast<float2*>(stage + (g + 8) * kProbsLd + col) =
                        make_float2(fast_ex2(s[nt][2] - m[1]) * l[1], fast_ex2(s[nt][3] - m[1]) * l[1]);
                }
                __syncwarp();
                const int nrows = min(16, S - qrow0);
                float* out = probs + ((static_cast<long long>(b) * A + h) * S + qrow0) * S + kb * kBlk;
                for (int r = 0; r < nrows; ++r) {
                    if (lane < kvalid) out[static_cast<long long>(r) * S + lane] = stage[r * kProbsLd + lane];
                    if (lane + 32 < kvalid) out[static_cast<long long>(r) * S + lane + 32] = stage[r * kProbsLd + lane + 32];
                }
                __syncwarp();  // the staging tile is rewritten by the next key block
            }
        }
        __syncthreads();  // every warp is done with ring slot (step & 1) before step + 2 loads into it
    }
}

static size_t probs_smem(int S) {
    const int nkb = (S + kBlk - 1) / kBlk;
    return 3 * kTileBytes + (4 * 16 * kProbsLd + nkb * kBlk) * sizeof(float);
}

int attn_probs(const void* qkv, const float* mask_bias, float* probs, int B, int S, int A, int H, cudaStream_t st) {
    VB_REQUIRE(B > 0 && S > 0 && A > 0, "attention: empty problem");
    VB_REQUIRE(H == A * kHd, "attention: head_dim must be 64 (hidden=%d heads=%d)", H, A);
    VB_REQUIRE(A <= 65535 && B <= 65535, "attention: grid too large");
    VB_REQUIRE(qkv != nullptr && mask_bias != nullptr && probs != nullptr, "attention probs: null pointer");
    VB_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0, "attention: qkv must be 16-byte aligned");
    const size_t smem = probs_smem(S);
    VB_REQUIRE(smem <= 227 * 1024, "attention probs: seq %d too long", S);
    static int configured[kMaxDevices] = {0};
    VB_CHECK_CUDA(ensure_dyn_smem(attn_probs_kernel, static_cast<int>(smem), configured));
    const dim3 grid((S + kBlk - 1) / kBlk, A, B);
    {
        ProfScope ps(st, PROF_ATTN_FWD, 2.0 * B * A * S * S * kHd, 1);
        VB_CHECK_CUDA(launch_pdl(attn_probs_kernel, grid, dim3(128), smem, st, static_cast<const bf16*>(qkv), mask_bias, probs, S,
                                 A, H));
    }
    return 0;
}

}  // namespace vb

extern "C" {
int vb_attention_probs(const void* qkv, const float* mask_bias, float* probs, int32_t batch, int32_t seq, int32_t heads,
                       int32_t hidden, void* stream) {
    return vb::attn_probs(qkv, mask_bias, probs, batch, seq, heads, hidden, static_cast<cudaStream_t>(stream));
}
}
