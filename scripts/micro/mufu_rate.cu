// Micro-benchmark: sustained MUFU.EX2 throughput per SM (and with an FFMA/ISETP mix like the render loop).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o mufu_rate mufu_rate.cu
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ float ex2(float x) { float y; asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
template <int MODE>
__global__ void k(float* out, int iters, float seed) {
    float a0 = seed + threadIdx.x * 1e-3f, a1 = a0 + 1.f, a2 = a0 + 2.f, a3 = a0 + 3.f;
    float s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    for (int i = 0; i < iters; ++i) {
        if (MODE == 0) {            // pure MUFU, 4 independent chains
            a0 = ex2(a0) - 1.0f; a1 = ex2(a1) - 1.0f; a2 = ex2(a2) - 1.0f; a3 = ex2(a3) - 1.0f;
        } else {                    // render-like mix: per MUFU 2 FFMA + 1 ISETP + 1 predicated FFMA + 1 FADD
            float q0 = fmaf(a0, a1, s0), q1 = fmaf(a1, a2, s1), q2 = fmaf(a2, a3, s2), q3 = fmaf(a3, a0, s3);
            q0 = fmaf(q0, a0, 0.5f); q1 = fmaf(q1, a1, 0.5f); q2 = fmaf(q2, a2, 0.5f); q3 = fmaf(q3, a3, 0.5f);
            float e0 = ex2(-q0), e1 = ex2(-q1), e2 = ex2(-q2), e3 = ex2(-q3);
            if (__float_as_uint(q0) < 0x42000000u) s0 = fmaf(e0, 0.3f, s0);
            if (__float_as_uint(q1) < 0x42000000u) s1 = fmaf(e1, 0.3f, s1);
            if (__float_as_uint(q2) < 0x42000000u) s2 = fmaf(e2, 0.3f, s2);
            if (__float_as_uint(q3) < 0x42000000u) s3 = fmaf(e3, 0.3f, s3);
            a0 += 1e-6f; a1 -= 1e-6f; a2 += 1e-6f; a3 -= 1e-6f;
        }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + s0 + s1 + s2 + s3;
}
int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount; float* out; cudaMalloc(&out, sms * 8 * 256 * 4);
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    for (int mode = 0; mode < 2; ++mode) for (int bps : {2, 4, 8}) {
        const int iters = 20000;
        cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
        if (mode == 0) k<0><<<sms * bps, 256>>>(out, 100, 0.1f); else k<1><<<sms * bps, 256>>>(out, 100, 0.1f);
        cudaEventRecord(a);
        if (mode == 0) k<0><<<sms * bps, 256>>>(out, iters, 0.1f); else k<1><<<sms * bps, 256>>>(out, iters, 0.1f);
        cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b);
        double mufu = (double)sms * bps * 256 * iters * 4;
        printf("mode %d, %d CTAs/SM: %.3f ms, %.2f MUFU lane-ops/ns total, %.2f per SM per clk @%d MHz nominal\n", mode, bps, ms,
               mufu / (ms * 1e6), mufu / (ms * 1e-3) / sms / (clk * 1e3), clk / 1000);
    }
    return 0;
}
