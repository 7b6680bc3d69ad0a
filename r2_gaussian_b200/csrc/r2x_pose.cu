// r2x_pose.cu -- per-view pose corrections on the device (r2x_pose_apply / r2x_pose_grad, include/r2x.h).
// The map is the one `pose.PoseCorrection.matrices` states with torch ops:
//   D      = exp([omega_i, nu_i]) - I           (Rodrigues + the SE(3) left Jacobian, series below theta^2 = 1e-2)
//   view'  = view + view D^T                    (view = T^T, so view' = (exp(xi) T)^T)
//   full'  = full + (view D^T) proj
// evaluated in float64 and rounded to float32 once per entry; a zero increment is taken as -0.0 so that a zero twist
// returns the camera's matrices bit for bit (x + -0.0 == x for every x, including -0.0).  The gradient is the exact
// chain rule through the same float64 expression: forward-mode dual numbers, one thread per twist direction.
// Both launches are tiny (one warp, resp. one warp plus the zero fill of the other rows) and read no host state.
#include <cmath>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {
namespace {

// value and derivative along one direction
struct Dual {
    double v, d;
    __device__ Dual(double x = 0.0, double dx = 0.0) : v(x), d(dx) {}
};
__device__ inline Dual operator+(Dual a, Dual b) { return Dual(a.v + b.v, a.d + b.d); }
__device__ inline Dual operator-(Dual a, Dual b) { return Dual(a.v - b.v, a.d - b.d); }
__device__ inline Dual operator-(Dual a) { return Dual(-a.v, -a.d); }
__device__ inline Dual operator*(Dual a, Dual b) { return Dual(a.v * b.v, a.d * b.v + a.v * b.d); }
__device__ inline Dual operator/(Dual a, Dual b) { return Dual(a.v / b.v, (a.d * b.v - a.v * b.d) / (b.v * b.v)); }
__device__ inline Dual sqrt(Dual a) {
    const double s = ::sqrt(a.v);
    return Dual(s, a.d / (2.0 * s));
}
__device__ inline Dual sin(Dual a) { return Dual(::sin(a.v), ::cos(a.v) * a.d); }
__device__ inline Dual cos(Dual a) { return Dual(::cos(a.v), -::sin(a.v) * a.d); }
__device__ inline double sqrt(double a) { return ::sqrt(a); }
__device__ inline double sin(double a) { return ::sin(a); }
__device__ inline double cos(double a) { return ::cos(a); }
__device__ inline double value(Dual a) { return a.v; }
__device__ inline double value(double a) { return a; }

// d_view = view (exp(xi) - I)^T and d_full = d_view proj, all [4,4] row-major as the torch tensors store them
template <typename T>
__device__ void pose_increments(const T w[3], const T n[3], const float* __restrict__ view,
                                const float* __restrict__ proj, T d_view[16], T d_full[16]) {
    const T K[3][3] = {{T(0.0), -w[2], w[1]}, {w[2], T(0.0), -w[0]}, {-w[1], w[0], T(0.0)}};
    T K2[3][3];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) K2[r][c] = K[r][0] * K[0][c] + K[r][1] * K[1][c] + K[r][2] * K[2][c];
    // pose._coefficients: a = sin t / t, b = (1 - cos t) / t^2, c = (t - sin t) / t^3, Taylor series below 1e-2
    const T x = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    T a, b, c;
    if (value(x) < 1e-2) {
        a = T(1.0) - x / T(6.0) * (T(1.0) - x / T(20.0) * (T(1.0) - x / T(42.0)));
        b = T(0.5) - x / T(24.0) * (T(1.0) - x / T(30.0) * (T(1.0) - x / T(56.0)));
        c = T(1.0 / 6) - x / T(120.0) * (T(1.0) - x / T(42.0) * (T(1.0) - x / T(72.0)));
    } else {
        const T t = sqrt(x), s = sin(t), co = cos(t);
        a = s / t;
        b = (T(1.0) - co) / x;
        c = (t - s) / (x * t);
    }
    T D[4][4];
    for (int r = 0; r < 3; ++r) {
        for (int c2 = 0; c2 < 3; ++c2) D[r][c2] = a * K[r][c2] + b * K2[r][c2];   // R - I
        T tr = n[r];                                                             // V nu, V = I + b K + c K^2
        for (int k = 0; k < 3; ++k) tr = tr + (b * K[r][k] + c * K2[r][k]) * n[k];
        D[r][3] = tr;
    }
    for (int c2 = 0; c2 < 4; ++c2) D[3][c2] = T(0.0);
    for (int r = 0; r < 4; ++r)
        for (int c2 = 0; c2 < 4; ++c2) {
            T s = T(0.0);
            for (int k = 0; k < 4; ++k) s = s + T((double)view[r * 4 + k]) * D[c2][k];
            d_view[r * 4 + c2] = s;
        }
    for (int r = 0; r < 4; ++r)
        for (int c2 = 0; c2 < 4; ++c2) {
            T s = T(0.0);
            for (int k = 0; k < 4; ++k) s = s + d_view[r * 4 + k] * T((double)proj[k * 4 + c2]);
            d_full[r * 4 + c2] = s;
        }
}

__device__ inline float add_increment(float base, double d) { return (float)((double)base + (d == 0.0 ? -0.0 : d)); }

// one warp: every lane forms the increments (a few hundred flops), lanes 0-15 write view', 16-31 full'
__global__ void __launch_bounds__(32) pose_apply_kernel(const float* __restrict__ omega, const float* __restrict__ nu,
                                                        int i, const float* __restrict__ view,
                                                        const float* __restrict__ full, const float* __restrict__ proj,
                                                        float* __restrict__ out_view, float* __restrict__ out_full) {
    const double w[3] = {omega[3 * i], omega[3 * i + 1], omega[3 * i + 2]};
    const double n[3] = {nu[3 * i], nu[3 * i + 1], nu[3 * i + 2]};
    double dv[16], df[16];
    pose_increments<double>(w, n, view, proj, dv, df);
    const int l = threadIdx.x;
    if (l < 16) out_view[l] = add_increment(view[l], dv[l]);
    else out_full[l - 16] = add_increment(full[l - 16], df[l - 16]);
}

// block 0, lanes 0-5: d loss / d xi_k of view i along direction k (omega 0-2, nu 3-5); every other entry of both
// outputs (other views, the anchor) is written 0
__global__ void __launch_bounds__(256) pose_grad_kernel(const float* __restrict__ omega, const float* __restrict__ nu,
                                                        int n_views, int i, int anchor, const float* __restrict__ view,
                                                        const float* __restrict__ proj, const float* __restrict__ gview,
                                                        const float* __restrict__ gproj, float* __restrict__ g_omega,
                                                        float* __restrict__ g_nu) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < 6 * n_views) {
        const int row = (e % (3 * n_views)) / 3;
        if (row != i || row == anchor) (e < 3 * n_views ? g_omega : g_nu)[e % (3 * n_views)] = 0.f;
    }
    if (blockIdx.x != 0 || threadIdx.x >= 6 || i == anchor) return;
    const int k = threadIdx.x;
    Dual w[3], n[3];
    for (int j = 0; j < 3; ++j) {
        w[j] = Dual(omega[3 * i + j], k == j ? 1.0 : 0.0);
        n[j] = Dual(nu[3 * i + j], k == 3 + j ? 1.0 : 0.0);
    }
    Dual dv[16], df[16];
    pose_increments<Dual>(w, n, view, proj, dv, df);
    double g = 0.0;
    for (int j = 0; j < 16; ++j) g += (double)gview[j] * dv[j].d + (double)gproj[j] * df[j].d;
    (k < 3 ? g_omega : g_nu)[3 * i + k % 3] = (float)g;
}

}  // namespace
}  // namespace r2x

extern "C" {

int r2x_pose_apply(void* stream, const float* omega, const float* nu, int n_views, int view_index,
                   const float* world_view_transform, const float* full_proj_transform, const float* projection_matrix,
                   float* out_world_view_transform, float* out_full_proj_transform) {
    using namespace r2x;
    if (!omega || !nu || !world_view_transform || !full_proj_transform || !projection_matrix ||
        !out_world_view_transform || !out_full_proj_transform)
        return fail_msg(R2X_ERR_INVALID, "r2x_pose_apply: null pointer");
    if (n_views <= 0) return fail_msg(R2X_ERR_INVALID, "r2x_pose_apply: n_views must be positive");
    if (view_index < 0 || view_index >= n_views) return fail_msg(R2X_ERR_INVALID, "r2x_pose_apply: view index out of range");
    pose_apply_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(omega, nu, view_index, world_view_transform,
                                                          full_proj_transform, projection_matrix,
                                                          out_world_view_transform, out_full_proj_transform);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

int r2x_pose_grad(void* stream, const float* omega, const float* nu, int n_views, int view_index, int anchor,
                  const float* world_view_transform, const float* projection_matrix, const float* dL_dview,
                  const float* dL_dproj, float* dL_domega, float* dL_dnu) {
    using namespace r2x;
    if (!omega || !nu || !world_view_transform || !projection_matrix || !dL_dview || !dL_dproj || !dL_domega ||
        !dL_dnu)
        return fail_msg(R2X_ERR_INVALID, "r2x_pose_grad: null pointer");
    if (n_views <= 0 || n_views > (1 << 26)) return fail_msg(R2X_ERR_INVALID, "r2x_pose_grad: n_views out of range");
    if (view_index < 0 || view_index >= n_views) return fail_msg(R2X_ERR_INVALID, "r2x_pose_grad: view index out of range");
    if (anchor < -1 || anchor >= n_views) return fail_msg(R2X_ERR_INVALID, "r2x_pose_grad: anchor index out of range");
    const int nblk = (6 * n_views + 255) / 256;
    pose_grad_kernel<<<nblk, 256, 0, (cudaStream_t)stream>>>(omega, nu, n_views, view_index, anchor,
                                                             world_view_transform, projection_matrix, dL_dview,
                                                             dL_dproj, dL_domega, dL_dnu);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
