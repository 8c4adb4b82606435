// Microbenchmark: peak throughput of warp-level mma.sync.m16n8k16 (bf16 -> fp32) on this GPU, as a function of
// resident warps per SM and independent accumulators per warp. Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3
#include <cstdio>
#include <cuda_runtime.h>
template <int ACC>
__global__ void k(float* out, int iters) {
    float c[ACC][4];
    for (int i = 0; i < ACC; ++i) c[i][0] = c[i][1] = c[i][2] = c[i][3] = 0.f;
    unsigned a0 = threadIdx.x, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, b0 = a0 * 3, b1 = a0 * 5;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < ACC; ++i)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(c[i][0]), "+f"(c[i][1]), "+f"(c[i][2]), "+f"(c[i][3])
                         : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    }
    float s = 0;
    for (int i = 0; i < ACC; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
    if (s == 12345.f) out[0] = s;
}
template <int ACC>
void run(int warps_per_sm) {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    float* d; cudaMalloc(&d, 4);
    const int iters = 20000, threads = 128, blocks = sms * warps_per_sm / 4;
    k<ACC><<<blocks, threads>>>(d, 100);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0); k<ACC><<<blocks, threads>>>(d, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double flops = 2.0 * 16 * 8 * 16 * (double)ACC * iters * blocks * 4;
    printf("acc=%d warps/SM=%2d: %.1f TFLOP/s\n", ACC, warps_per_sm, flops / ms / 1e9);
    cudaFree(d);
}
int main() {
    for (int w : {4, 8, 12, 16, 32}) { run<1>(w); run<2>(w); run<4>(w); run<8>(w); }
    return 0;
}
