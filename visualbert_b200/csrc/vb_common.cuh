// vb_common.cuh — sm_90a device primitives shared by every kernel in libvbert_b200.
//
// Thin inline-PTX wrappers (mbarrier, TMA, wgmma) plus small math helpers.
// No CUTLASS/CuTe dependency: the descriptors are built by hand (see vb_gemm.cu).
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

namespace vb {

typedef __nv_bfloat16 bf16;

// host-side shared state / helpers (defined in vb_gemm.cu)
extern std::atomic<long long> g_launches;  // kernel launches issued by this library
int num_sms();      // SM count of the CALLER'S CURRENT device (cached per device)
constexpr int kMaxDevices = 64;
int current_device();  // cudaGetDevice, clamped to [0, kMaxDevices)
// Deterministic reductions (vb_set_deterministic): the calling thread's workspace, ptr == nullptr when the mode is off.
struct DetWs { void* ptr; long long bytes; };
DetWs det_ws();
// 0 when the mode is off or `need` bytes fit the workspace; else sets the error (naming the bytes) and returns 2
int det_require(long long need, const char* what);
// Device-side dropout seed offset (vb_set_dropout_offset): the calling thread's uint64 device pointer, nullptr when unset. While
// it is set, every launch that draws dropout bits runs the kernel instantiation that adds *offset to its seed when it runs.
const unsigned long long* drop_offset();
// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device property of a kernel: `cache` is the caller's static
// per-device record of the size already configured (DataParallel threads / several devices in one process).
template <typename K>
inline cudaError_t ensure_dyn_smem(K kern, int bytes, int (&cache)[kMaxDevices]) {
    const int d = current_device();
    if (cache[d] >= bytes) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) cache[d] = bytes;
    return e;
}

// Optional live profiling (vb_profile_enable): every launcher brackets its kernels with CUDA events on
// the launch stream and tags them with a category and the algorithmic work (FLOPs or bytes) of the call.
enum { PROF_GEMM_FWD = 0, PROF_GEMM_DGRAD = 1, PROF_GEMM_WGRAD = 2, PROF_ATTN_FWD = 3, PROF_ATTN_DQ = 4, PROF_ATTN_DKV = 5,
       PROF_LN_FWD = 6, PROF_LN_BWD = 7, PROF_COLSUM = 8, PROF_EMBED = 9, PROF_OTHER = 10, PROF_NCAT = 11 };
// ---- programmatic dependent launch (PDL) -------------------------------------------------------------------
// Hot-path kernels are launched with cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel's CTAs may be
// scheduled, and run their on-chip prologue (barrier init, tensor-map prefetch), while the previous
// kernel's last CTAs drain. Every such kernel calls pdl_trigger() on entry and pdl_wait() BEFORE its first global
// memory access (griddepcontrol.wait returns once the preceding grid has completed and its writes are visible).
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

struct ProfScope {
    ProfScope(cudaStream_t st, int cat, double work, int launches);
    ~ProfScope();
    int slot;
    cudaStream_t st;
};

// ---------------------------------------------------------------------------------------------
// error plumbing (host)
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
#define VB_CHECK_CUDA(expr)                                                                   \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            vb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return 1;                                                                         \
        }                                                                                     \
    } while (0)
#define VB_REQUIRE(cond, ...)                                                                 \
    do {                                                                                      \
        if (!(cond)) {                                                                        \
            vb::set_error(__VA_ARGS__);                                                       \
            return 2;                                                                         \
        }                                                                                     \
    } while (0)

#define VB_TRY_RC(expr)      \
    do {                     \
        int _rc = (expr);    \
        if (_rc) return _rc; \
    } while (0)

// true when every pointer is 16-byte aligned (NULL counts as aligned): what a kernel that moves 16-byte vectors needs of the
// pointers it is handed, checked by its entry point before the first CUDA call
template <typename... T>
inline bool all_aligned16(const T*... p) {
    return ((reinterpret_cast<uintptr_t>(p) | ... | uintptr_t{0}) & 15) == 0;
}

// ---------------------------------------------------------------------------------------------
// generic helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t v) {
    __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&v);
    return __bfloat1622float2(h);
}

// raw SFU approximations (1 MUFU each, no range fix-up branches); ex2(-inf) = +0
__device__ __forceinline__ float fast_ex2(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_rcp(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// gelu(x) = x * 0.5 * (1 + erf(x / sqrt(2)))   — reference modeling.py:56-61 (exact-erf form).
// erf via Abramowitz-Stegun 7.1.26 (|abs err| < 1.5e-7 + SFU approximation error ~1e-6, far below the
// bf16 output rounding): erf(|z|) = 1 - (a1 t + ... + a5 t^5) exp(-z^2), t = 1 / (1 + p |z|).
// Returns q = poly(t) * t * exp(-x^2/2) so that erf(|x|/sqrt2) = 1 - q; also hands back exp(-x^2/2).
__device__ __forceinline__ float erfc_abs_sqrt2(float x, float& e) {
    const float ax = fabsf(x);
    e = fast_ex2(x * x * -0.72134752044448170f);              // exp(-x^2/2)
    const float t = fast_rcp(fmaf(0.23164189f, ax, 1.0f));    // p/sqrt(2) = 0.3275911 * 0.70710678
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    return poly * t * e;
}
__device__ __forceinline__ float gelu_fwd(float x) {
    float e;
    const float q = erfc_abs_sqrt2(x, e);
    const float hx = 0.5f * x, ha = fabsf(hx);
    return fmaf(-ha, q, hx + ha);  // 0.5 x + 0.5 |x| (1 - q)
}
// gelu(x) and d/dx gelu(x) = Phi(x) + x phi(x) from the same exp / rcp (the FFN-up epilogue stores both, so the
// backward epilogue is a single multiply)
__device__ __forceinline__ void gelu_fwd_bwd(float x, float& g, float& gp) {
    float e;
    const float q = erfc_abs_sqrt2(x, e);
    const float cdf = 0.5f + copysignf(fmaf(-0.5f, q, 0.5f), x);
    g = x * cdf;
    gp = fmaf(x * e, 0.3989422804014327f, cdf);
}
// d/dx gelu(x) = 0.5 (1 + erf(x/√2)) + x φ(x),  φ(x) = exp(-x²/2)/√(2π)
__device__ __forceinline__ float gelu_bwd(float x) {
    float e;
    const float q = erfc_abs_sqrt2(x, e);
    const float cdf = 0.5f + copysignf(fmaf(-0.5f, q, 0.5f), x);
    return fmaf(x * e, 0.3989422804014327f, cdf);
}

// ---------------------------------------------------------------------------------------------
// counter-based dropout RNG: a pure function of (seed, stream id, element index), so forward and
// backward regenerate the same keep-mask without storing it. One 32-bit avalanche hash (lowbias32
// finaliser, ~8 integer ops) yields two 16-bit uniforms, i.e. 4 ops per element — the epilogues that
// apply dropout are ALU-bound, a 10-round Philox (13 ops per element) measurably slowed them down.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du;
    x ^= x >> 15; x *= 0x846ca68bu;
    x ^= x >> 16;
    return x;
}
__device__ __forceinline__ uint32_t dropout_key(uint64_t seed, uint32_t stream) {
    return mix32(static_cast<uint32_t>(seed) ^ mix32(static_cast<uint32_t>(seed >> 32) + 0x9E3779B9u * (stream + 1u)));
}
// Hidden-state dropout quantises the drop probability to n/256 (0.1 -> 26/256 = 0.1016) and scales survivors by
// 256/(256-n), so E[dropout(x)] = x exactly while one hash serves 4 elements and the threshold test is a single
// SIMD byte compare. Host side: dropout_quantise().
struct DropQ { unsigned thr8; float scale; };
inline DropQ dropout_quantise(float p) {
    DropQ q;
    unsigned n = static_cast<unsigned>(p * 256.0f + 0.5f);
    if (n > 255u) n = 255u;
    q.thr8 = n;
    q.scale = p > 0.f ? 256.0f / (256.0f - static_cast<float>(n)) : 0.f;
    return q;
}
// Keep-mask bits for the 8 consecutive elements starting at flat element index `elem8 * 8`.
// Each element consumes 8 random bits; kept iff bits >= thr8. dropout_keep8_key takes key0 = dropout_key(seed, stream).
__device__ __forceinline__ uint32_t dropout_keep8_key(uint32_t key0, uint64_t elem8, uint32_t thr8) {
    const uint32_t key = key0 ^ (static_cast<uint32_t>(elem8 >> 31) * 0x27d4eb2fu);
    const uint32_t base = static_cast<uint32_t>(elem8) << 1;
    const uint32_t t4 = thr8 * 0x01010101u;
    // __vcmpgeu4: per-byte (a >= b) ? 0xff : 0x00; the multiply gathers the 4 byte LSBs into one nibble
    const uint32_t m0 = __vcmpgeu4(mix32(base ^ key), t4) & 0x01010101u;
    const uint32_t m1 = __vcmpgeu4(mix32((base + 1u) ^ key), t4) & 0x01010101u;
    return ((m0 * 0x01020408u) >> 24) | (((m1 * 0x01020408u) >> 24) << 4);
}
__device__ __forceinline__ uint32_t dropout_keep8(uint64_t seed, uint32_t stream, uint64_t elem8, uint32_t thr8) {
    return dropout_keep8_key(dropout_key(seed, stream), elem8, thr8);
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (the kernel fails with an error the host reports) instead of hanging the GPU:
// ~4e9 cycles ≈ 2 s at 1.9 GHz, far beyond any legitimate wait in these kernels. Kept tiny and fully inline — the
// hot kernels wait at dozens of sites (code size = instruction-cache misses on every role switch), and a shared
// out-of-line helper would make ptxas apply the SMALLEST setmaxnreg budget of its callers to all of them.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0x3ffu) == 0 && clock64() - t0 > 4000000000ll) __trap();
    }
}

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) — 2-D tiled load, completion on an mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar,
                                            int c_inner, int c_outer) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c_inner), "r"(c_outer)
        : "memory");
}

// 2-D tiled store shared -> global (bulk-group completion); the box is clipped at the tensor's bounds
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t smem_src, int c_inner, int c_outer) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_src), "r"(c_inner), "r"(c_outer)
                 : "memory");
}
// contiguous bulk copies (16-byte aligned addresses, size a multiple of 16)
__device__ __forceinline__ void bulk_load(uint32_t smem_dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void bulk_store(void* dst, uint32_t smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(reinterpret_cast<uint64_t>(dst)), "r"(smem_src), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the shared-memory sources of every committed bulk store have been read (the global writes may still be in flight)
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// Four 8 x 8 bf16 matrices between shared memory and the wgmma accumulator fragment: lane l addresses row l % 8 of matrix l / 8,
// register k holds the pair (row l / 4, columns 2 (l % 4), +1) of matrix k.
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr)
                 : "memory");
}
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3])
                 : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a)
// ---------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle: start address, leading / stride byte offsets (16-byte units).
//  K-major  tile [rows][64]: 8-row groups are 1024 B apart (SBO); LBO unused.
//  MN-major tile [atoms of 64 along MN][64 k-rows][64]: 8 k-rows = 1024 B (SBO), next 64-wide MN atom = 8192 B (LBO).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4) | (static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           (static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 128] (+)= A[64 x 16] * B[16 x 128], bf16 in, fp32 accumulators in registers of the warpgroup.
// TA / TB = 1: the operand is MN-major in shared memory (transposed read), 0: K-major.
// Fragment of thread t (warp w = t / 32, lane l): d[4 j + 2 i + c] = D[16 w + l / 4 + 8 i][8 j + 2 (l % 4) + c].
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, %67, %68;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB));
}
// D[64 x 256] (+)= A[64 x 16] * B[16 x 256]: one instruction for a 256-wide tile reads the A slice once (two m64n128k16 read it
// twice). Fragment as above with j = 0..31: d[4 j + 2 i + c] = D[16 w + l / 4 + 8 i][8 j + 2 (l % 4) + c].
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, %131, %132;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB));
}
// D[64 x 64] (+)= A[64 x 16] * B[16 x 64], both operands from shared-memory descriptors (fragment of D as above).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, %35, %36;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB));
}
// same with A from registers: a[0..3] of thread (warp w, lane l) hold the bf16 pairs (16 w + l/4, 2 (l%4)), (+8 rows, same cols),
// (same row, +8 cols), (+8 rows, +8 cols) — the accumulator layout of a 64 x 16 slice, so a result feeds the next MMA directly.
template <int TB>
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, %38;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate), "n"(TB));
}
// One lane of a CONVERGED warp (elect.sync): the producer loop runs with all 32 lanes converged and only the issue is
// predicated, so loop state stays in uniform registers.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "elect.sync _|P1, 0xffffffff;\n"
        "selp.u32 %0, 1, 0, P1;\n"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}
// Register re-distribution between warp roles (whole warpgroups of 4 warps): the producer warpgroup shrinks its
// allocation, the MMA warpgroups grow theirs; ptxas compiles the code that follows against the new limit.
template <int N>
__device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------------------------------------
// vectorised global access
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_v4(const void* p) {
    return __ldg(reinterpret_cast<const uint4*>(p));
}
__device__ __forceinline__ void stg_v4(void* p, uint4 v) { *reinterpret_cast<uint4*>(p) = v; }
// 32 bytes per thread as two 128-bit accesses (one full 32-byte sector)
__device__ __forceinline__ void ldg_v8(const void* p, uint32_t (&r)[8]) {
    const uint4 a = ldg_v4(p), b = ldg_v4(static_cast<const uint8_t*>(p) + 16);
    r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}
__device__ __forceinline__ void stg_v8(void* p, const uint32_t (&r)[8]) {
    stg_v4(p, make_uint4(r[0], r[1], r[2], r[3]));
    stg_v4(static_cast<uint8_t*>(p) + 16, make_uint4(r[4], r[5], r[6], r[7]));
}
__device__ __forceinline__ void red_add_v4_f32(float* p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c),
                 "f"(d)
                 : "memory");
}

}  // namespace vb
