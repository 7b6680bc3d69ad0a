// r2x_compact.cu -- device-side stream compaction for densify / clone / split / prune (SURVEY.md 8(f) rank 3).
//
// The reference rebuilds its 4 parameter tensors, their 8 Adam moment tensors and its per-Gaussian statistics with
// boolean-mask indexing and torch.cat, several times per densification step (gaussian_model.py:335-403, :503-550):
// every `t[mask]` is a nonzero() + gather with a host synchronisation.  Here a row selection is built ONCE:
//
//   r2x_mask_select   mask[n] (bytes)  ->  stable list of the selected row indices + their count (on the device):
//                     mask -> 0/1 words -> single-pass decoupled-look-back scan -> scatter.  No host round trip;
//                     the caller reads the count when it needs the new row count (one read per densification step).
//   r2x_gather_rows   ONE launch gathers every per-Gaussian tensor (parameters, both Adam moments, statistics) through
//                     that list.  A source is the virtual concatenation [src0 (n0 rows) | src1]; src1 == NULL means
//                     "zeros" (the Adam moments / statistics of freshly created rows).
#include "../../include/r2x.h"
#include "r2x_binning.cuh"

namespace r2x {

__global__ void mask_words_kernel(int n, const unsigned char* __restrict__ mask, uint32_t* __restrict__ words) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) words[i] = mask[i] ? 1u : 0u;
}

__global__ void mask_scatter_kernel(int n, const unsigned char* __restrict__ mask, const uint32_t* __restrict__ incl,
                                    int* __restrict__ idx_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && mask[i]) idx_out[incl[i] - 1u] = i;
}

struct GatherPack {
    r2x_gather_desc d[R2X_GATHER_MAX_TENSORS];
    int n;
};

__global__ void __launch_bounds__(256) gather_rows_kernel(GatherPack pk, const int* __restrict__ select, long long nsel) {
    const r2x_gather_desc d = pk.d[blockIdx.y];
    const long long total = nsel * d.width;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long row = e / d.width;
        const int col = (int)(e - row * d.width);
        const long long src = select ? (long long)select[row] : row;
        float v = 0.f;
        if (src < d.n0) v = d.src0[src * d.width + col];
        else if (d.src1) v = d.src1[(src - d.n0) * d.width + col];
        d.dst[e] = v;
    }
}

size_t mask_select_scratch_bytes(int n) {
    const size_t m = (size_t)(n > 0 ? n : 1);
    return ((m * 4 + 255) / 256 * 256) * 2 + ((scan_state_bytes((int)m) + 255) / 256 * 256) + 256;
}

int launch_mask_select(cudaStream_t st, int n, const unsigned char* mask, int* idx_out, uint32_t* count_dev,
                       void* scratch, size_t scratch_bytes) {
    if (n < 0 || !count_dev) return fail_msg(R2X_ERR_INVALID, "r2x_mask_select: bad arguments");
    if (n == 0) {
        R2X_CUDA_OK(cudaMemsetAsync(count_dev, 0, sizeof(uint32_t), st));
        return 0;
    }
    if (!mask || !idx_out || !scratch || scratch_bytes < mask_select_scratch_bytes(n))
        return fail_msg(R2X_ERR_INVALID, "r2x_mask_select: null pointer / scratch too small");
    const size_t per = ((size_t)n * 4 + 255) / 256 * 256;
    char* p = (char*)(((size_t)scratch + 255) / 256 * 256);
    uint32_t* words = (uint32_t*)p; p += per;
    uint32_t* incl = (uint32_t*)p; p += per;
    void* state = p;
    mask_words_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, mask, words);
    R2X_CUDA_OK(cudaGetLastError());
    const int rc = launch_scan(st, n, words, incl, state, count_dev);
    if (rc) return rc;
    mask_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, mask, incl, idx_out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_gather_rows(cudaStream_t st, int ntensors, const r2x_gather_desc* descs, const int* select, long long nsel) {
    if (ntensors < 0 || ntensors > R2X_GATHER_MAX_TENSORS) return fail_msg(R2X_ERR_INVALID, "r2x_gather_rows: too many tensors");
    if (nsel < 0) return fail_msg(R2X_ERR_INVALID, "r2x_gather_rows: negative row count");
    if (ntensors == 0 || nsel == 0) return 0;
    if (!descs) return fail_msg(R2X_ERR_INVALID, "r2x_gather_rows: null descriptors");
    GatherPack pk{};
    pk.n = ntensors;
    long long widest = 1;
    for (int i = 0; i < ntensors; ++i) {
        pk.d[i] = descs[i];
        if (descs[i].width <= 0 || descs[i].n0 < 0 || !descs[i].dst || (descs[i].n0 > 0 && !descs[i].src0))
            return fail_msg(R2X_ERR_INVALID, "r2x_gather_rows: bad descriptor");
        if (descs[i].width > widest) widest = descs[i].width;
    }
    long long nb = (nsel * widest + 255) / 256;
    int sms;
    R2X_CUDA_OK(sm_count(&sms));
    if (nb > sms * 8) nb = sms * 8;
    gather_rows_kernel<<<dim3((unsigned)nb, (unsigned)ntensors), 256, 0, st>>>(pk, select, nsel);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace r2x

extern "C" {

size_t r2x_mask_select_scratch_bytes(int n) { return r2x::mask_select_scratch_bytes(n); }

int r2x_mask_select(void* stream, int n, const unsigned char* mask, int* idx_out, uint32_t* count_dev, void* scratch,
                    size_t scratch_bytes) {
    return r2x::launch_mask_select((cudaStream_t)stream, n, mask, idx_out, count_dev, scratch, scratch_bytes);
}

int r2x_gather_rows(void* stream, int ntensors, const r2x_gather_desc* descs, const int* select, long long nsel) {
    return r2x::launch_gather_rows((cudaStream_t)stream, ntensors, descs, select, nsel);
}

}  // extern "C"
