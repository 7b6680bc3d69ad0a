// r2x_common.cuh -- shared device helpers for the sm_90a X-ray Gaussian kernels.
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#include "r2x_matcalc.cuh"

#define R2X_TILE 16     // detector tile edge, pixels   (reference RAS/config.h:16-17)
#define R2X_VTILE 8     // voxel tile edge              (reference VOX/config.h:16-18)

#define R2X_CUDA_OK(expr)                                                      \
    do {                                                                       \
        cudaError_t _e = (expr);                                               \
        if (_e != cudaSuccess) return r2x::fail(_e, #expr, __FILE__, __LINE__); \
    } while (0)

namespace r2x {

int fail(cudaError_t e, const char* what, const char* file, int line);
int fail_msg(int code, const char* msg);
// Streaming multiprocessors of the current device (132 on an H100 SXM), queried once per device: persistent and
// grid-stride launches size their grids from it.  A failed query is returned as an error, never guessed.
cudaError_t sm_count(int* n);

// ---------------------------------------------------------------------------------------------
// Folded parameter activations (SURVEY 8(f) rank 2; the reference applies them as separate torch kernels,
// gaussian_model.py:112-126): with `enabled` the preprocess kernels read the RAW parameters and apply
//     density = softplus(raw)              (torch.nn.Softplus: x > 20 ? x : log1p(exp(x)))
//     scale   = lo + (hi - lo) sigmoid(raw)   [scale_mode 1]   or   exp(raw)   [scale_mode 0]
//     rotation = raw / max(|raw|, 1e-12)   (torch.nn.functional.normalize)
// themselves, and the per-Gaussian backward kernels return the gradients with respect to the raw parameters.
// ---------------------------------------------------------------------------------------------
struct Activation {
    int enabled;
    int scale_mode;
    float lo, hi;
};
Activation current_activation();                 // set by the *_raw entry points for the duration of one call (r2x_api.cu)
void set_activation(const Activation* a);

__device__ __forceinline__ float act_softplus(float x) { return x > 20.0f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float act_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float act_scale(const Activation& a, float x) {
    return a.scale_mode ? __fadd_rn(__fmul_rn(act_sigmoid(x), a.hi - a.lo), a.lo) : expf(x);
}
__device__ __forceinline__ float act_scale_grad(const Activation& a, float x) {   // d scale / d raw
    if (!a.scale_mode) return expf(x);
    const float sg = act_sigmoid(x);
    return (a.hi - a.lo) * sg * (1.0f - sg);
}
// norm receives the unclamped |q|
__device__ __forceinline__ float4 act_normalize(float4 q, float& norm) {
    norm = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    const float inv = 1.0f / fmaxf(norm, 1e-12f);
    return make_float4(q.x * inv, q.y * inv, q.z * inv, q.w * inv);
}
// gradient of q_hat = q / max(|q|, 1e-12) pulled back to q:  (dq_hat - q_hat (q_hat . dq_hat)) / |q|; below the clamp
// the denominator is a constant (torch's clamp_min passes no gradient to |q|), so the gradient is dq_hat / 1e-12
__device__ __forceinline__ void act_normalize_grad(float4 qn, float norm, float* dr) {
    const float dot = norm >= 1e-12f ? qn.x * dr[0] + qn.y * dr[1] + qn.z * dr[2] + qn.w * dr[3] : 0.0f;
    const float inv = 1.0f / fmaxf(norm, 1e-12f);
    dr[0] = (dr[0] - qn.x * dot) * inv; dr[1] = (dr[1] - qn.y * dot) * inv;
    dr[2] = (dr[2] - qn.z * dot) * inv; dr[3] = (dr[3] - qn.w * dot) * inv;
}

// ---------------------------------------------------------------------------------------------
// Exactly-rounded float32 building blocks.  The reference's radii / tile rectangles / depth bits
// must be reproduced bit for bit, so every operation on that path is written with an explicit
// rounding intrinsic: the compiler can neither fuse nor re-associate them.  The sequence mirrors
// the FMA contraction nvcc chose for the reference's own expressions (DESIGN.md section 3).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float frcp(float a) { return __frcp_rn(a); }
__device__ __forceinline__ float fsqrt(float a) { return __fsqrt_rn(a); }

// a0*b0 + a1*b1 + a2*b2  ==  fma(a2,b2, fma(a0,b0, rn(a1*b1)))
__device__ __forceinline__ float dot3c(float a0, float b0, float a1, float b1, float a2, float b2) {
    return ffma(a2, b2, ffma(a0, b0, fmul(a1, b1)));
}
// row r of a column-major-flat 4x4 applied to (x,y,z,1)
__device__ __forceinline__ float xform_row(const float* __restrict__ m, int r, float x, float y, float z) {
    return fadd(m[12 + r], ffma(z, m[8 + r], ffma(x, m[r], fmul(y, m[4 + r]))));
}

// Sigma = (S R)^T (S R) from scale*mod and the un-normalised quaternion (r,x,y,z);
// six floats (S00,S01,S02,S11,S12,S22).
__device__ __forceinline__ void cov3d_from_scale_rot(float s0, float s1, float s2, float mod, float4 q, float* cov) {
    const float sx = fmul(mod, s0), sy = fmul(mod, s1), sz = fmul(mod, s2);
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    // (SASS-level contraction of the reference build: r*x, r*z, x*z, y*y, z*z are rounded products,
    //  every other product rides inside an FMA)
    const float yy = fmul(y, y), zz = fmul(z, z), xz = fmul(x, z), rx = fmul(r, x), rz = fmul(r, z);
    const float yy_zz = fadd(yy, zz);
    const float xx_zz = ffma(x, x, zz);
    const float xx_yy = ffma(x, x, yy);
    const float a02 = ffma(r, y, xz), a20 = ffma(-r, y, xz);
    const float a12 = ffma(y, z, -rx), a21 = ffma(y, z, rx);
    const float a01 = ffma(x, y, -rz), a10 = ffma(x, y, rz);
    const float R00 = fsub(1.0f, fadd(yy_zz, yy_zz));
    const float R01 = fadd(a01, a01), R02 = fadd(a02, a02), R10 = fadd(a10, a10);
    const float R11 = fsub(1.0f, fadd(xx_zz, xx_zz));
    const float R12 = fadd(a12, a12), R20 = fadd(a20, a20), R21 = fadd(a21, a21);
    const float R22 = fsub(1.0f, fadd(xx_yy, xx_yy));
    const float M00 = fmul(sx, R00), M01 = fmul(sy, R01), M02 = fmul(sz, R02);
    const float M10 = fmul(sx, R10), M11 = fmul(sy, R11), M12 = fmul(sz, R12);
    const float M20 = fmul(sx, R20), M21 = fmul(sy, R21), M22 = fmul(sz, R22);
    cov[0] = dot3c(M00, M00, M01, M01, M02, M02);
    cov[1] = dot3c(M10, M00, M11, M01, M12, M02);
    cov[2] = dot3c(M20, M00, M21, M01, M22, M02);
    cov[3] = dot3c(M10, M10, M11, M11, M12, M12);
    cov[4] = dot3c(M20, M10, M21, M11, M22, M12);
    cov[5] = dot3c(M20, M20, M21, M21, M22, M22);
}

// ---------------------------------------------------------------------------------------------
// TMA (1-D bulk async copy) + mbarrier helpers.  SASS: UBLKCP / SYNCS.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// non-blocking: has the phase with this parity completed?
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// global -> shared bulk copy; bytes multiple of 16, both addresses 16-byte aligned.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// 16-byte Ampere-style async gather (LDGSTS): per-thread source address.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
// the mbarrier receives one (pre-counted) arrival when all cp.async copies this thread issued so far have landed
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Programmatic dependent launch (sm_90+): a kernel launched through pdl_launch() may become resident while its
// predecessor in the stream is still running; it parks in pdl_wait() until that predecessor has completed and its
// writes are visible, so the launch latency and the CTA ramp of every kernel of a forward / backward chain overlap
// the tail of the previous one.  Every kernel launched this way calls pdl_prologue() before touching global memory
// (inputs may be outputs of the predecessor, outputs may still be read by it) and thereby lets its own successor in.
__device__ __forceinline__ void pdl_prologue() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
template <typename... KArgs, typename... Args>
inline cudaError_t pdl_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    static int enabled = -1;          // R2X_NO_PDL=1: plain stream-ordered launches (measurement of what PDL buys)
    if (enabled < 0) {
        const char* e = getenv("R2X_NO_PDL");
        enabled = (e && e[0] == '1') ? 0 : 1;
    }
    cfg.numAttrs = enabled ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// FP32 pairs carried in one 64-bit register pair.  Hopper has no packed FP32 arithmetic, so each operation is two
// scalar FMUL / FADD / FFMA with the same round-to-nearest, no-flush semantics per lane; pack2 / unpack2 are register
// renames that the compiler removes.
__device__ __forceinline__ uint64_t pack2(float a, float b) {
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ void unpack2(uint64_t v, float& a, float& b) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
    float a0, a1, b0, b1;
    unpack2(a, a0, a1); unpack2(b, b0, b1);
    return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t add2(uint64_t a, uint64_t b) {
    float a0, a1, b0, b1;
    unpack2(a, a0, a1); unpack2(b, b0, b1);
    return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
    float a0, a1, b0, b1, c0, c1;
    unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
    return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

}  // namespace r2x
