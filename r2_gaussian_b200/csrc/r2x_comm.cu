// One-shot all-reduce (sum) of a small tensor over NVLink peer memory: the exchange step of the Gaussian-sharded
// projector (every rank renders its shard of the Gaussians into its own partial image; the detector image is the
// sum over ranks).  Replaces `dist.all_reduce` (NCCL: ~35-40 us for 1 MiB on 8 GPUs, latency bound) by one kernel:
//
//   1. tell every peer "my partial image of step `epoch` is complete" (a release store into the peer's flag array);
//   2. wait until every peer said the same (acquire loads of the local flag array);
//   3. read all `world` partial images -- the peers' through NVLink, 128-bit loads -- and add them IN RANK ORDER, so
//      every rank ends up with the same bits, run to run (NCCL's ring / tree order is not specified).
//
// Buffers live in cudaMalloc memory shared through CUDA IPC handles (peer access enabled lazily by the open call).
// Partial images are double-buffered by the caller (epoch parity): a rank may overwrite a buffer two steps later,
// and by then every peer has signalled the step in between, i.e. has finished reading.
#include <cstdint>
#include <cstring>

#include "../../include/r2x.h"
#include "r2x_binning.cuh"
#include "r2x_common.cuh"

namespace r2x {

struct PeerPack {
    const float* buf[R2X_MAX_PEERS];
    uint32_t* flags[R2X_MAX_PEERS];
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 ld_volatile_f4(const float4* p) {
    float4 v;
    asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

__global__ void __launch_bounds__(256) peer_allreduce_kernel(PeerPack pk, int world, int rank, uint32_t epoch,
                                                             float* __restrict__ out, long long n,
                                                             uint32_t* __restrict__ status, long long timeout_cycles) {
    // 1. signal (one CTA), 2. wait (every CTA)
    if (blockIdx.x == 0 && threadIdx.x < world) st_release_sys(pk.flags[threadIdx.x] + rank, epoch);
    if (threadIdx.x < world) {
        const uint32_t* f = pk.flags[rank] + threadIdx.x;
        const long long t0 = clock64();
        while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) {
            if (clock64() - t0 > timeout_cycles) {   // a peer never arrived; report instead of hanging the GPU
                atomicExch(status, 1u);
                break;
            }
        }
    }
    __syncthreads();
    // 3. ordered sum.  All peer loads of an element are issued before the first add (the adds wait on the loads'
    //    scoreboards in program order: interleaving load/add would serialise the NVLink round trips).
    const long long n4 = n >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 v[R2X_MAX_PEERS];
#pragma unroll
        for (int p = 0; p < R2X_MAX_PEERS; ++p)
            if (p < world) v[p] = ld_volatile_f4(reinterpret_cast<const float4*>(pk.buf[p]) + i);
        float4 acc = v[0];
#pragma unroll
        for (int p = 1; p < R2X_MAX_PEERS; ++p)
            if (p < world) { acc.x += v[p].x; acc.y += v[p].y; acc.z += v[p].z; acc.w += v[p].w; }
        reinterpret_cast<float4*>(out)[i] = acc;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0)
        for (long long i = n4 << 2; i < n; ++i) {
            float acc = *reinterpret_cast<const volatile float*>(pk.buf[0] + i);
            for (int p = 1; p < world; ++p) acc += *reinterpret_cast<const volatile float*>(pk.buf[p] + i);
            out[i] = acc;
        }
}

int launch_peer_allreduce(cudaStream_t st, int world, int rank, const float* const* bufs, uint32_t* const* flags,
                          uint32_t epoch, float* out, long long n, uint32_t* status, long long timeout_cycles) {
    if (world < 1 || world > R2X_MAX_PEERS || rank < 0 || rank >= world)
        return fail_msg(R2X_ERR_INVALID, "r2x_peer_allreduce_sum: bad world/rank");
    if (!bufs || !flags || !out || !status || n < 0) return fail_msg(R2X_ERR_INVALID, "r2x_peer_allreduce_sum: null pointer");
    PeerPack pk{};
    for (int p = 0; p < world; ++p) {
        if (!bufs[p] || !flags[p]) return fail_msg(R2X_ERR_INVALID, "r2x_peer_allreduce_sum: null peer buffer");
        if (((size_t)bufs[p] & 15) != 0) return fail_msg(R2X_ERR_INVALID, "r2x_peer_allreduce_sum: buffers must be 16-byte aligned");
        pk.buf[p] = bufs[p];
        pk.flags[p] = flags[p];
    }
    if (((size_t)out & 15) != 0) return fail_msg(R2X_ERR_INVALID, "r2x_peer_allreduce_sum: out must be 16-byte aligned");
    long long nb = ((n >> 2) + 255) / 256;
    if (nb < 1) nb = 1;
    int sms;
    R2X_CUDA_OK(sm_count(&sms));
    if (nb > sms) nb = sms;     // all CTAs spin on the flags: keep the grid within one wave
    if (timeout_cycles <= 0) timeout_cycles = 1ll << 32;   // ~2 s
    peer_allreduce_kernel<<<(unsigned)nb, 256, 0, st>>>(pk, world, rank, epoch, out, n, status, timeout_cycles);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace r2x

extern "C" {

int r2x_peer_alloc(size_t bytes, void** dev_ptr) {
    if (!dev_ptr) return r2x::fail_msg(R2X_ERR_INVALID, "r2x_peer_alloc: null pointer");
    R2X_CUDA_OK(cudaMalloc(dev_ptr, bytes ? bytes : 1));
    R2X_CUDA_OK(cudaMemset(*dev_ptr, 0, bytes ? bytes : 1));
    R2X_CUDA_OK(cudaDeviceSynchronize());
    return 0;
}

int r2x_peer_free(void* dev_ptr) {
    if (dev_ptr) R2X_CUDA_OK(cudaFree(dev_ptr));
    return 0;
}

int r2x_ipc_export(void* dev_ptr, unsigned char* handle64) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
    if (!dev_ptr || !handle64) return r2x::fail_msg(R2X_ERR_INVALID, "r2x_ipc_export: null pointer");
    cudaIpcMemHandle_t h;
    R2X_CUDA_OK(cudaIpcGetMemHandle(&h, dev_ptr));
    memcpy(handle64, &h, 64);
    return 0;
}

int r2x_ipc_open(const unsigned char* handle64, void** dev_ptr) {
    if (!handle64 || !dev_ptr) return r2x::fail_msg(R2X_ERR_INVALID, "r2x_ipc_open: null pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    R2X_CUDA_OK(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}

int r2x_ipc_close(void* dev_ptr) {
    if (dev_ptr) R2X_CUDA_OK(cudaIpcCloseMemHandle(dev_ptr));
    return 0;
}

int r2x_peer_allreduce_sum(void* stream, int world, int rank, const float* const* bufs, uint32_t* const* flags,
                           uint32_t epoch, float* out, long long n, uint32_t* status_dev) {
    return r2x::launch_peer_allreduce((cudaStream_t)stream, world, rank, bufs, flags, epoch, out, n, status_dev, 0);
}

int r2x_peer_allreduce_sum_t(void* stream, int world, int rank, const float* const* bufs, uint32_t* const* flags,
                             uint32_t epoch, float* out, long long n, uint32_t* status_dev, long long timeout_cycles) {
    return r2x::launch_peer_allreduce((cudaStream_t)stream, world, rank, bufs, flags, epoch, out, n, status_dev,
                                      timeout_cycles);
}

}  // extern "C"
