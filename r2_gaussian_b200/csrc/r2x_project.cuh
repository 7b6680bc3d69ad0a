// r2x_project.cuh -- the per-ray setup of the volume projector, shared by the projector (r2x_project.cu) and its
// matched backprojector (r2x_backproject.cu), so that both see the same float32 sample positions by construction.
#pragma once

#include <cmath>
#include <cstdio>

namespace r2x {

// One detector pixel's ray in the volume's index space: sample k sits at p_k = fmaf(k, s, g) (lattice point i at
// p = i), for the integers k0 <= k <= k1 whose sample lies inside the field's support (-1, n) on every axis (cone beam
// also t > 0).  k0 > k1 when the ray misses the box.
struct ProjRay {
    float gx, gy, gz;   // g_c: the ray's closest approach to the volume centre
    float sx, sy, sz;   // index-space step
    long long k0, k1;
};

// The detector is offset by (tu, tv) pixels (TIGRE's geo.offDetector over its pixel pitch; 0, 0 when centred), so pixel
// (v, u) sees the ray of the centred detector's fractional pixel (v - tv, u + tu): ndc_x gains su = 2 tu / W and ndc_y
// loses sv = 2 tv / H (ProjShift, divided once on the host: IEEE division gives the same bits there).  Zero shifts add
// exact zeros, so a centred detector's rays are unchanged bit for bit.
struct ProjShift {
    double su, sv;
};

__host__ __device__ inline ProjShift proj_shift(float tu, float tv, int H, int W) {
    return {2.0 * (double)tu / W, 2.0 * (double)tv / H};
}

// Columns of a per-view geometry table row (include/r2x.h): float64 [N, VG_COLS].
constexpr int VG_COLS = 5, VG_TANX = 0, VG_TANY = 1, VG_SHIFT_U = 2, VG_SHIFT_V = 3, VG_DSO = 4;

// Host check of a per-view geometry table (the host copy of the device table the kernels read) before any CUDA work:
// present, every value finite once rounded to float32 as the kernels round it, tan_fov > 0 (cone beam, or always when
// `tan_always`), dso > 0 in cone beam.  Returns 0 or the fail_msg code.
static inline int view_geometry_check(const char* who, int N, int mode, const double* dev, const double* host,
                                      bool tan_always) {
    char msg[192];
    if (!dev || !host) {
        std::snprintf(msg, sizeof msg, "%s: bad pointer (view_geometry NULL)", who);
        return fail_msg(R2X_ERR_INVALID, msg);
    }
    for (int v = 0; v < N; ++v) {
        const double* row = host + (size_t)v * VG_COLS;
        const char* bad = nullptr;
        for (int c = 0; c < VG_COLS; ++c)
            if (!std::isfinite((float)row[c])) bad = "values must be finite";
        if (!bad && (mode == 1 || tan_always) && !((float)row[VG_TANX] > 0.0f && (float)row[VG_TANY] > 0.0f))
            bad = "tan_fov must be > 0";
        if (!bad && mode == 1 && !((float)row[VG_DSO] > 0.0f)) bad = "cone beam needs dso > 0";
        if (bad) {
            std::snprintf(msg, sizeof msg, "%s: bad view_geometry (view %d: %s)", who, v, bad);
            return fail_msg(R2X_ERR_INVALID, msg);
        }
    }
    return 0;
}

// TABLE: the view's tan_fov and shift come from its row of the per-view geometry table `vg` (include/r2x.h), rounded
// to float32 as the scalar entry points' arguments are, so a view is bit for bit the scalar call with its values.
// Without TABLE, `vg` is not read and the code is the scalar setup's.
template <bool CONE, bool TABLE>
__device__ __forceinline__ ProjRay project_ray_setup(const float* __restrict__ viewm, int view, int u, int v, int H,
                                                     int W, int nx, int ny, int nz, float sx, float sy, float sz,
                                                     float cx, float cy, float cz, float tanx, float tany,
                                                     float step, ProjShift shift,
                                                     const double* __restrict__ vg) {
    if (TABLE) {
        const double* row = vg + (size_t)view * VG_COLS;
        tanx = (float)row[VG_TANX];
        tany = (float)row[VG_TANY];
        shift = proj_shift((float)row[VG_SHIFT_U], (float)row[VG_SHIFT_V], H, W);
    }
    // world -> camera: rotation Rw[r][c] = m[4c + r], translation T[r] = m[12 + r] (column-major flat)
    const float* m = viewm + (size_t)view * 16;
    double Rw[3][3], T[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) Rw[r][c] = (double)__ldg(m + 4 * c + r);
        T[r] = (double)__ldg(m + 12 + r);
    }
    // camera-frame ray of the pixel centre: cone from the source, parallel from (ndc_x, ndc_y, 0), both along +z
    double ndx = (2.0 * u + 1.0) / W - 1.0, ndy = (2.0 * v + 1.0) / H - 1.0;
    ndx += shift.su;
    ndy -= shift.sv;
    const double oc[3] = {CONE ? 0.0 : ndx, CONE ? 0.0 : ndy, 0.0};
    const double dc[3] = {CONE ? ndx * (double)tanx : 0.0, CONE ? ndy * (double)tany : 0.0, 1.0};
    // to world through the rigid inverse (Rw^T, -Rw^T T), relative to the volume centre
    const double ctr[3] = {(double)cx, (double)cy, (double)cz};
    double o[3], d[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        o[c] = Rw[0][c] * (oc[0] - T[0]) + Rw[1][c] * (oc[1] - T[1]) + Rw[2][c] * (oc[2] - T[2]) - ctr[c];
        d[c] = Rw[0][c] * dc[0] + Rw[1][c] * dc[1] + Rw[2][c] * dc[2];
    }
    const double inv_len = 1.0 / sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    d[0] *= inv_len; d[1] *= inv_len; d[2] *= inv_len;
    const double tc = -(o[0] * d[0] + o[1] * d[1] + o[2] * d[2]);   // closest approach to the volume centre
    // index space: lattice point i (voxel centre) at g = i; the field is nonzero only for g in (-1, n)
    const int n[3] = {nx, ny, nz};
    const double s[3] = {(double)sx, (double)sy, (double)sz};
    double g[3], st[3];
    double lo = -1e300, hi = 1e300;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double dv = s[a] / n[a];
        g[a] = (o[a] + tc * d[a]) / dv + 0.5 * (n[a] - 1);
        st[a] = (double)step * d[a] / dv;
        if (st[a] != 0.0) {
            const double k1 = (-1.0 - g[a]) / st[a], k2 = ((double)n[a] - g[a]) / st[a];
            lo = fmax(lo, fmin(k1, k2));
            hi = fmin(hi, fmax(k1, k2));
        } else if (!(g[a] > -1.0 && g[a] < (double)n[a])) {
            lo = 1.0; hi = 0.0;                                        // parallel to this slab and outside it
        }
    }
    ProjRay r;
    r.k0 = (long long)ceil(fmax(lo, -1e18));
    r.k1 = (long long)floor(fmin(hi, 1e18));
    if (CONE) r.k0 = max(r.k0, (long long)floor(fmin(fmax(-tc / (double)step, -1e18), 1e18)) + 1);   // t > 0
    r.gx = (float)g[0]; r.gy = (float)g[1]; r.gz = (float)g[2];
    r.sx = (float)st[0]; r.sy = (float)st[1]; r.sz = (float)st[2];
    return r;
}

}  // namespace r2x
