/*
 * r2_oracle.c -- CPU restatement of the R2-Gaussian X-ray rasterizer and voxelizer.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (r2_gaussian_b200/,
 * xray_gaussian_rasterization_voxelization/) may import, link or execute this
 * file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs use it, as the checker / CPU baseline.
 *
 * Parity pinning: the reference ships NO golden vectors or tests for this
 * path (SURVEY.md section 4).  This restatement is pinned instead against the
 * reference's own CUDA sources compiled for sm_90a into oracle/_ref/
 * (oracle/build_ref.sh, with oracle/glm_standin standing in for the
 * un-vendored GLM submodule) and run on the GPU, whose outputs are stored under
 * tests/golden/ref/: tests/test_ref_gpu.py compares them with the oracle bit-exactly on radii / tiles_touched / sort keys and
 * to 1e-5 on intensities, and tests/golden/ holds vectors produced by that
 * reference build (tests/golden/make_golden.py).
 *
 * Bit-exact territory (radii, tile rectangles, depth bits -> sort keys): the
 * float32 dataflow below reproduces, operation by operation, the FMA
 * contraction nvcc 12.9 chose for the reference's expressions (read from
 * `nvcc -ptx` of the reference sources):  a*b + c*d + e*f is evaluated as
 * fma(e,f, fma(a,b, round(c*d))), `x + bias` after such a dot as a separate
 * add, ndc2Pix and mu in float64.  This file must be compiled with
 * -ffp-contract=off so the C compiler does not add contractions of its own.
 *
 * Each function cites the reference file:line it follows
 * (RAS = r2_gaussian/submodules/xray-gaussian-rasterization-voxelization/cuda_rasterizer,
 *  VOX = .../cuda_voxelizer).
 */
#define _GNU_SOURCE
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define TILE_X 16 /* RAS/config.h:16-17 */
#define TILE_Y 16
#define VT 8 /* VOX/config.h:16-18 */

/* ----------------------------------------------------------------------------
 * helpers
 * -------------------------------------------------------------------------- */

/* a0*b0 + a1*b1 + a2*b2 as nvcc contracted it: fma(a2,b2, fma(a0,b0, a1*b1)) */
static inline float dot3c(float a0, float b0, float a1, float b1, float a2, float b2) {
    float m = a1 * b1;
    return fmaf(a2, b2, fmaf(a0, b0, m));
}

/* RAS/auxiliary.h:62-81 transformPoint4x3/4x4 row r: m[r]*x + m[4+r]*y + m[8+r]*z + m[12+r] */
static inline float xform_row(const float* m, int r, float x, float y, float z) {
    float t = y * m[4 + r];
    t = fmaf(x, m[r], t);
    t = fmaf(z, m[8 + r], t);
    return m[12 + r] + t;
}

static inline uint32_t f2u(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
}

static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* RAS/forward.cu:161-195 (identical copy at VOX/forward.cu:21-55): Sigma = (S R)^T (S R),
 * quaternion (r,x,y,z) consumed un-normalised; stored (S00,S01,S02,S11,S12,S22). */
static void cov3d_from_scale_rot(const float* scale, float mod, const float* q, float* cov) {
    float sx = mod * scale[0], sy = mod * scale[1], sz = mod * scale[2];
    float r = q[0], x = q[1], y = q[2], z = q[3];
    /* SASS-level contraction (ptxas fuses further than the PTX shows): the products r*x, r*z, x*z and
     * y*y, z*z are rounded; every other product of the rotation entries rides inside an FMA. */
    float yy = y * y, zz = z * z, xz = x * z, rx = r * x, rz = r * z;
    float yy_zz = yy + zz;
    float xx_zz = fmaf(x, x, zz);
    float xx_yy = fmaf(x, x, yy);
    float ry_xz = fmaf(r, y, xz);    /* x*z + r*y */
    float xz_ry = fmaf(-r, y, xz);   /* x*z - r*y */
    float yz_rx_m = fmaf(y, z, -rx); /* y*z - r*x */
    float yz_rx_p = fmaf(y, z, rx);  /* y*z + r*x */
    float xy_rz_m = fmaf(x, y, -rz); /* x*y - r*z */
    float xy_rz_p = fmaf(x, y, rz);  /* x*y + r*z */
    /* textual rows of R in the reference; glm columns */
    float R00 = 1.0f - (yy_zz + yy_zz);
    float R01 = xy_rz_m + xy_rz_m;
    float R02 = ry_xz + ry_xz;
    float R10 = xy_rz_p + xy_rz_p;
    float R11 = 1.0f - (xx_zz + xx_zz);
    float R12 = yz_rx_m + yz_rx_m;
    float R20 = xz_ry + xz_ry;
    float R21 = yz_rx_p + yz_rx_p;
    float R22 = 1.0f - (xx_yy + xx_yy);
    /* M = S * R (glm):  M[c][r] = s_r * Rcol[c][r]; Rcol[0]=(R00,R01,R02) ... */
    float M00 = sx * R00, M01 = sy * R01, M02 = sz * R02;
    float M10 = sx * R10, M11 = sy * R11, M12 = sz * R12;
    float M20 = sx * R20, M21 = sy * R21, M22 = sz * R22;
    /* Sigma[c][r] = sum_k M[r][k] * M[c][k] */
    cov[0] = dot3c(M00, M00, M01, M01, M02, M02);
    cov[1] = dot3c(M10, M00, M11, M01, M12, M02);
    cov[2] = dot3c(M20, M00, M21, M01, M22, M02);
    cov[3] = dot3c(M10, M10, M11, M11, M12, M12);
    cov[4] = dot3c(M20, M10, M21, M11, M22, M12);
    cov[5] = dot3c(M20, M20, M21, M21, M22, M22);
}

/* The 3x3 world->ray-space matrix M = W * J of RAS/forward.cu:85-123, as 9 floats
 * Mm[c*3+r] = M[c][r] (glm column c, row r), plus the clamped view-space point t. */
static void raster_build_M(const float* mean, const float* view, float focal_x, float focal_y,
                           float tan_fovx, float tan_fovy, int mode, float* Mm, float* t_out,
                           float* txtz_out, float* tytz_out) {
    float tx = xform_row(view, 0, mean[0], mean[1], mean[2]);
    float ty = xform_row(view, 1, mean[0], mean[1], mean[2]);
    float tz = xform_row(view, 2, mean[0], mean[1], mean[2]);
    float J00, J02, J11, J12, J20, J21, J22;
    if (mode == 0) { /* parallel beam: RAS/forward.cu:87-98 (t.x,t.y clamp is dead code) */
        J00 = focal_x; J02 = 0.f; J11 = focal_y; J12 = 0.f; J20 = 0.f; J21 = 0.f; J22 = 1.f;
        if (txtz_out) { *txtz_out = tx; *tytz_out = ty; }
        float lim = 1.3f;
        tx = fminf(lim, fmaxf(-lim, tx));
        ty = fminf(lim, fmaxf(-lim, ty));
    } else { /* cone beam: RAS/forward.cu:99-115 */
        float limx = tan_fovx * 1.3f, limy = tan_fovy * 1.3f;
        float txtz = tx / tz, tytz = ty / tz;
        if (txtz_out) { *txtz_out = txtz; *tytz_out = tytz; }
        tx = tz * fminf(limx, fmaxf(-limx, txtz));
        ty = tz * fminf(limy, fmaxf(-limy, tytz));
        float tz2 = tz * tz;
        float l = sqrtf(tz2 + fmaf(tx, tx, ty * ty));
        J00 = focal_x / tz;
        J02 = (focal_x * (-tx)) / tz2;
        J11 = focal_y / tz;
        J12 = (focal_y * (-ty)) / tz2;
        J20 = tx / l; J21 = ty / l; J22 = tz / l;
    }
    /* W[k][r] = view[k + 4r];  M[c][r] = W[0][r]*J[c][0] + W[1][r]*J[c][1] + W[2][r]*J[c][2]
     * with glm columns J[0]=(J00,0,J02), J[1]=(0,J11,J12), J[2]=(J20,J21,J22). */
    for (int r = 0; r < 3; ++r) {
        float w0 = view[4 * r], w1 = view[4 * r + 1], w2 = view[4 * r + 2];
        Mm[0 * 3 + r] = dot3c(w0, J00, w1, 0.f, w2, J02);
        Mm[1 * 3 + r] = dot3c(w0, 0.f, w1, J11, w2, J12);
        Mm[2 * 3 + r] = dot3c(w0, J20, w1, J21, w2, J22);
    }
    t_out[0] = tx; t_out[1] = ty; t_out[2] = tz;
}

/* cov = M^T * Vrk^T * M, RAS/forward.cu:125-131; returns the six entries
 * hat = (cov00, cov01, cov02, cov11, cov12, cov22). */
static void raster_cov_from_M(const float* Mm, const float* c3, float* hat) {
    float T[9]; /* T[c*3+r] = (M^T Vrk^T)[c][r] = sum_k M[r][k] * Vrk[k][c] */
    const float V[9] = {c3[0], c3[1], c3[2], c3[1], c3[3], c3[4], c3[2], c3[4], c3[5]};
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r)
            T[c * 3 + r] = dot3c(Mm[r * 3 + 0], V[c * 3 + 0], Mm[r * 3 + 1], V[c * 3 + 1], Mm[r * 3 + 2], V[c * 3 + 2]);
    /* cov[c][r] = sum_k T[k][r] * M[c][k] */
#define COV(c, r) dot3c(T[0 * 3 + (r)], Mm[(c) * 3 + 0], T[1 * 3 + (r)], Mm[(c) * 3 + 1], T[2 * 3 + (r)], Mm[(c) * 3 + 2])
    hat[0] = COV(0, 0) + 0.0f;
    hat[1] = COV(0, 1);
    hat[2] = COV(0, 2);
    hat[3] = COV(1, 1) + 0.0f;
    hat[4] = COV(1, 2);
    hat[5] = COV(2, 2);
#undef COV
}

/* circ = det3 of the ray-space covariance exactly as contracted for RAS/forward.cu:148 */
static inline float det3_ref(float a, float b, float c, float d, float e, float f, float ad) {
    float t = ad * f;
    t = fmaf((b + b) * c, e, t);
    t = fmaf(-e, a * e, t);
    t = fmaf(-b, b * f, t);
    t = fmaf(-c, c * d, t);
    return t;
}

/* ----------------------------------------------------------------------------
 * Rasterizer forward: per-Gaussian preprocess (RAS/forward.cu:198-289)
 * Outputs (all length-P arrays): radii, xy[2P], depth, cov3D[6P], conic_opacity[4P],
 * mu, tiles_touched, rect[4P]=(xmin,ymin,xmax,ymax).  Returns sum(tiles_touched).
 * -------------------------------------------------------------------------- */
long long orc_raster_preprocess(int P, const float* means, const float* scales, float scale_modifier,
                                const float* rots, const float* opac, const float* cov3D_precomp,
                                const float* view, const float* proj, int W, int H, float tan_fovx,
                                float tan_fovy, int mode, int* radii, float* xy, float* depth,
                                float* cov3D, float* conic_opacity, float* mu, uint32_t* tiles_touched,
                                int* rect) {
    const float focal_y = H / (2.0f * tan_fovy); /* RAS/rasterizer_impl.cu:219-220 */
    const float focal_x = W / (2.0f * tan_fovx);
    const int gx = (W + TILE_X - 1) / TILE_X, gy = (H + TILE_Y - 1) / TILE_Y;
    long long total = 0;
#pragma omp parallel for reduction(+ : total) schedule(static)
    for (int i = 0; i < P; ++i) {
        radii[i] = 0;
        tiles_touched[i] = 0;
        xy[2 * i] = xy[2 * i + 1] = 0.f;
        depth[i] = 0.f;
        mu[i] = 0.f;
        for (int k = 0; k < 4; ++k) { conic_opacity[4 * i + k] = 0.f; rect[4 * i + k] = 0; }
        const float* p = means + 3 * i;
        /* in_frustum, RAS/auxiliary.h:143-168: only the near cull z_view <= 0.2 */
        float zv = xform_row(view, 2, p[0], p[1], p[2]);
        if (zv <= 0.2f) continue;
        float hx = xform_row(proj, 0, p[0], p[1], p[2]);
        float hy = xform_row(proj, 1, p[0], p[1], p[2]);
        float hw = xform_row(proj, 3, p[0], p[1], p[2]);
        float pw = 1.0f / (hw + 0.0000001f);
        float px = hx * pw, py = hy * pw;
        const float* c3;
        if (cov3D_precomp) {
            c3 = cov3D_precomp + 6 * i;
            if (cov3D) memcpy(cov3D + 6 * i, c3, 24);
        } else {
            cov3d_from_scale_rot(scales + 3 * i, scale_modifier, rots + 4 * i, cov3D + 6 * i);
            c3 = cov3D + 6 * i;
        }
        float Mm[9], t[3], hat[6];
        raster_build_M(p, view, focal_x, focal_y, tan_fovx, tan_fovy, mode, Mm, t, NULL, NULL);
        raster_cov_from_M(Mm, c3, hat);
        float a = hat[0], b = hat[1], c = hat[2], d = hat[3], e = hat[4], f = hat[5];
        float ad = a * d;
        float det = fmaf(-b, b, ad); /* diamond, RAS/forward.cu:147 == det, :261 */
        float circ = det3_ref(a, b, c, d, e, f, ad);
        if (det == 0.0f) continue;
        float det_inv = 1.0f / det;
        float conx = d * det_inv, cony = det_inv * (-b), conz = a * det_inv;
        float mid = (a + d) * 0.5f;
        float disc = sqrtf(fmaxf(fmaf(mid, mid, -det), 0.1f));
        float lam = fmaxf(mid + disc, mid - disc);
        float my_radius = ceilf(sqrtf(lam) * 3.0f);
        /* ndc2Pix in float64, RAS/auxiliary.h:45-48 */
        float pix_x = (float)(fma((double)px + 1.0, (double)W, -1.0) * 0.5);
        float pix_y = (float)(fma((double)py + 1.0, (double)H, -1.0) * 0.5);
        /* getRect, RAS/auxiliary.h:50-60 */
        int ri = (int)my_radius;
        float rf = (float)ri;
        int x0 = imin(gx, imax(0, (int)((pix_x - rf) * 0.0625f)));
        int y0 = imin(gy, imax(0, (int)((pix_y - rf) * 0.0625f)));
        int x1 = imin(gx, imax(0, (int)((((pix_x + rf) + 16.0f) + -1.0f) * 0.0625f)));
        int y1 = imin(gy, imax(0, (int)((((pix_y + rf) + 16.0f) + -1.0f) * 0.0625f)));
        int nt = (x1 - x0) * (y1 - y0);
        if (nt == 0) continue;
        /* mu, RAS/forward.cu:149-153 (float64 island) */
        double musq = ((double)circ * 6.283185307179586) / (double)det;
        float muv = ((float)musq > 0.0f) ? (float)sqrt(musq) : 0.0f;
        depth[i] = zv;
        radii[i] = ri;
        xy[2 * i] = pix_x;
        xy[2 * i + 1] = pix_y;
        conic_opacity[4 * i + 0] = conx;
        conic_opacity[4 * i + 1] = cony;
        conic_opacity[4 * i + 2] = conz;
        conic_opacity[4 * i + 3] = opac[i];
        mu[i] = muv;
        tiles_touched[i] = (uint32_t)nt;
        rect[4 * i + 0] = x0; rect[4 * i + 1] = y0; rect[4 * i + 2] = x1; rect[4 * i + 3] = y1;
        total += nt;
    }
    return total;
}

/* duplicateWithKeys, RAS/rasterizer_impl.cu:70-111 (VOX/voxelizer_impl.cu:54-101 for the 3-D
 * cube): emits (tile<<32 | depth_bits, gaussian id) row-major over the rectangle, Gaussians in
 * index order.  rect has 4 ints per Gaussian (2-D) or 6 (3-D: x0,y0,z0,x1,y1,z1). */
void orc_emit_keys(int P, int dims, const int* rect, const uint32_t* tiles_touched, const float* depth,
                   int gx, int gy, uint64_t* keys, uint32_t* vals) {
    size_t off = 0;
    for (int i = 0; i < P; ++i) {
        if (!tiles_touched[i]) continue;
        uint64_t db = f2u(depth[i]);
        if (dims == 2) {
            const int* r = rect + 4 * i;
            for (int y = r[1]; y < r[3]; ++y)
                for (int x = r[0]; x < r[2]; ++x) {
                    keys[off] = ((uint64_t)(uint32_t)(y * gx + x) << 32) | db;
                    vals[off++] = (uint32_t)i;
                }
        } else {
            const int* r = rect + 6 * i;
            for (int z = r[2]; z < r[5]; ++z)
                for (int y = r[1]; y < r[4]; ++y)
                    for (int x = r[0]; x < r[3]; ++x) {
                        keys[off] = ((uint64_t)(uint32_t)(z * gy * gx + y * gx + x) << 32) | db;
                        vals[off++] = (uint32_t)i;
                    }
        }
    }
}

/* Stable sort of (key,value) pairs == cub::DeviceRadixSort::SortPairs over all significant
 * bits (RAS/rasterizer_impl.cu:298-306), then identifyTileRanges (:116-138). LSD radix, 16 bits/pass. */
void orc_sort_pairs(size_t n, uint64_t* keys, uint32_t* vals) {
    if (n == 0) return;
    uint64_t* k2 = (uint64_t*)malloc(n * sizeof(uint64_t));
    uint32_t* v2 = (uint32_t*)malloc(n * sizeof(uint32_t));
    size_t* cnt = (size_t*)malloc(65537 * sizeof(size_t));
    uint64_t *ks = keys, *kd = k2;
    uint32_t *vs = vals, *vd = v2;
    for (int pass = 0; pass < 4; ++pass) {
        int sh = 16 * pass;
        memset(cnt, 0, 65537 * sizeof(size_t));
        for (size_t i = 0; i < n; ++i) cnt[((ks[i] >> sh) & 0xFFFF) + 1]++;
        for (int b = 0; b < 65536; ++b) cnt[b + 1] += cnt[b];
        for (size_t i = 0; i < n; ++i) {
            size_t d = cnt[(ks[i] >> sh) & 0xFFFF]++;
            kd[d] = ks[i];
            vd[d] = vs[i];
        }
        uint64_t* tk = ks; ks = kd; kd = tk;
        uint32_t* tv = vs; vs = vd; vd = tv;
    }
    /* 4 passes: data is back in the caller's arrays */
    free(k2); free(v2); free(cnt);
}

void orc_tile_ranges(size_t n, const uint64_t* keys, int ntiles, uint32_t* ranges /* 2*ntiles */) {
    memset(ranges, 0, (size_t)ntiles * 2 * sizeof(uint32_t));
    for (size_t i = 0; i < n; ++i) {
        uint32_t cur = (uint32_t)(keys[i] >> 32);
        if (i == 0) ranges[2 * cur] = 0;
        else {
            uint32_t prev = (uint32_t)(keys[i - 1] >> 32);
            if (cur != prev) { ranges[2 * prev + 1] = (uint32_t)i; ranges[2 * cur] = (uint32_t)i; }
        }
        if (i == n - 1) ranges[2 * cur + 1] = (uint32_t)n;
    }
}

/* renderCUDA forward, RAS/forward.cu:294-395: per pixel, walk the tile's list in sorted order;
 * power>0 or alpha<1e-5 pairs are skipped; plain float32 running sum in list order. */
void orc_raster_render(int W, int H, const uint32_t* ranges, const uint32_t* point_list, const float* xy,
                       const float* conic_opacity, const float* mu, float* out_color, uint32_t* n_contrib) {
    const int gx = (W + TILE_X - 1) / TILE_X, gy = (H + TILE_Y - 1) / TILE_Y;
#pragma omp parallel for schedule(dynamic, 1)
    for (int tile = 0; tile < gx * gy; ++tile) {
        int tx = tile % gx, ty = tile / gx;
        uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        for (int ly = 0; ly < TILE_Y; ++ly)
            for (int lx = 0; lx < TILE_X; ++lx) {
                int pxi = tx * TILE_X + lx, pyi = ty * TILE_Y + ly;
                if (pxi >= W || pyi >= H) continue;
                float pxf = (float)pxi, pyf = (float)pyi;
                float C = 0.f;
                uint32_t contributor = 0, last = 0;
                for (uint32_t s = r0; s < r1; ++s) {
                    uint32_t g = point_list[s];
                    contributor++;
                    float dx = xy[2 * g] - pxf, dy = xy[2 * g + 1] - pyf;
                    const float* co = conic_opacity + 4 * g;
                    /* -0.5f*(A dx dx + C dy dy) - B dx dy, contraction as in the reference PTX */
                    float q = fmaf(dx, dx * co[0], dy * (dy * co[2]));
                    float power = q * -0.5f - dy * (dx * co[1]);
                    if (power > 0.0f) continue;
                    float alpha = (co[3] * mu[g]) * expf(power);
                    if (alpha < 0.00001f) continue;
                    C += alpha;
                    last = contributor;
                }
                out_color[pyi * W + pxi] = C;
                if (n_contrib) n_contrib[pyi * W + pxi] = last;
            }
    }
}

/* Whole forward = Rasterizer::forward, RAS/rasterizer_impl.cu:196-331.  Caller provides
 * per-Gaussian outputs; keys/vals/ranges are returned through malloc'ed buffers the caller frees
 * with orc_free.  Returns num_rendered. */
long long orc_raster_forward(int P, const float* means, const float* scales, float scale_modifier,
                             const float* rots, const float* opac, const float* cov3D_precomp,
                             const float* view, const float* proj, int W, int H, float tan_fovx,
                             float tan_fovy, int mode, float* out_color, int* radii, float* xy,
                             float* depth, float* cov3D, float* conic_opacity, float* mu,
                             uint32_t* tiles_touched, int* rect, uint32_t* n_contrib,
                             uint64_t** keys_out, uint32_t** vals_out, uint32_t** ranges_out) {
    const int gx = (W + TILE_X - 1) / TILE_X, gy = (H + TILE_Y - 1) / TILE_Y;
    long long R = orc_raster_preprocess(P, means, scales, scale_modifier, rots, opac, cov3D_precomp, view, proj,
                                        W, H, tan_fovx, tan_fovy, mode, radii, xy, depth, cov3D, conic_opacity,
                                        mu, tiles_touched, rect);
    uint64_t* keys = (uint64_t*)malloc((size_t)(R > 0 ? R : 1) * sizeof(uint64_t));
    uint32_t* vals = (uint32_t*)malloc((size_t)(R > 0 ? R : 1) * sizeof(uint32_t));
    uint32_t* ranges = (uint32_t*)malloc((size_t)gx * gy * 2 * sizeof(uint32_t));
    orc_emit_keys(P, 2, rect, tiles_touched, depth, gx, gy, keys, vals);
    orc_sort_pairs((size_t)R, keys, vals);
    orc_tile_ranges((size_t)R, keys, gx * gy, ranges);
    orc_raster_render(W, H, ranges, vals, xy, conic_opacity, mu, out_color, n_contrib);
    if (keys_out) *keys_out = keys; else free(keys);
    if (vals_out) *vals_out = vals; else free(vals);
    if (ranges_out) *ranges_out = ranges; else free(ranges);
    return R;
}

void orc_free(void* p) { free(p); }

/* ----------------------------------------------------------------------------
 * Rasterizer backward
 * -------------------------------------------------------------------------- */

/* renderCUDA backward, RAS/backward.cu:447-575.  The reference accumulates each per-pair float32
 * term with float atomicAdd in nondeterministic order; the oracle forms each term in float32
 * exactly as the reference does and sums the terms in float64 (order-independent centre value),
 * rounding once at the end.  dL_dmean2D[3P] (x,y used), dL_dconic[4P] (x,y,.,w), dL_dopacity[P], dL_dmu[P]. */
void orc_raster_render_backward(int W, int H, int P, const uint32_t* ranges, const uint32_t* point_list,
                                const float* xy, const float* conic_opacity, const float* mu,
                                const float* dL_dpix, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                                float* dL_dmu) {
    const int gx = (W + TILE_X - 1) / TILE_X, gy = (H + TILE_Y - 1) / TILE_Y;
    double* acc = (double*)calloc((size_t)P * 7, sizeof(double));
    const float ddelx_dx = (float)(0.5 * W), ddely_dy = (float)(0.5 * H);
    for (int tile = 0; tile < gx * gy; ++tile) {
        int tx = tile % gx, ty = tile / gx;
        uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        for (int ly = 0; ly < TILE_Y; ++ly)
            for (int lx = 0; lx < TILE_X; ++lx) {
                int pxi = tx * TILE_X + lx, pyi = ty * TILE_Y + ly;
                if (pxi >= W || pyi >= H) continue;
                float pxf = (float)pxi, pyf = (float)pyi;
                float dLp = dL_dpix[pyi * W + pxi];
                for (uint32_t s = r0; s < r1; ++s) {
                    uint32_t g = point_list[s];
                    float dx = xy[2 * g] - pxf, dy = xy[2 * g + 1] - pyf;
                    const float* co = conic_opacity + 4 * g;
                    float q = fmaf(dx, dx * co[0], dy * (dy * co[2]));
                    float power = q * -0.5f - dy * (dx * co[1]);
                    if (power > 0.0f) continue;
                    float G = expf(power);
                    float m = mu[g];
                    float alpha = co[3] * m * G;
                    if (alpha < 0.00001f) continue;
                    float dL_dalpha = dLp;
                    float dL_dG = co[3] * m * dL_dalpha;
                    float gdx = G * dx, gdy = G * dy;
                    float dG_ddelx = -gdx * co[0] - gdy * co[1];
                    float dG_ddely = -gdy * co[2] - gdx * co[1];
                    double* a = acc + (size_t)g * 7;
                    a[0] += (double)(dL_dG * dG_ddelx * ddelx_dx);
                    a[1] += (double)(dL_dG * dG_ddely * ddely_dy);
                    a[2] += (double)(-0.5f * gdx * dx * dL_dG);
                    a[3] += (double)(-1.0f * gdx * dy * dL_dG);
                    a[4] += (double)(-0.5f * gdy * dy * dL_dG);
                    a[5] += (double)(m * G * dL_dalpha);
                    a[6] += (double)(co[3] * G * dL_dalpha);
                }
            }
    }
    for (int g = 0; g < P; ++g) {
        const double* a = acc + (size_t)g * 7;
        dL_dmean2D[3 * g + 0] = (float)a[0];
        dL_dmean2D[3 * g + 1] = (float)a[1];
        dL_dmean2D[3 * g + 2] = 0.f;
        dL_dconic[4 * g + 0] = (float)a[2];
        dL_dconic[4 * g + 1] = (float)a[3];
        dL_dconic[4 * g + 2] = 0.f;
        dL_dconic[4 * g + 3] = (float)a[4];
        dL_dopacity[g] = (float)a[5];
        dL_dmu[g] = (float)a[6];
    }
    free(acc);
}

/* computeCov3D backward, RAS/backward.cu:334-397 (same code VOX/backward.cu:21-84):
 * dL/dSigma(6) -> dL/dscale(3), dL/dquat(4) (no normalisation Jacobian). */
static void cov3d_backward(const float* scale, float mod, const float* q, const float* dL_dcov3D,
                           float* dL_dscale, float* dL_drot) {
    float r = q[0], x = q[1], y = q[2], z = q[3];
    /* textual rows of R (glm columns) */
    float Rc[3][3] = {
        {1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
        {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
        {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
    float s[3] = {mod * scale[0], mod * scale[1], mod * scale[2]};
    float M[3][3]; /* M = S*R : M[c][r] = s_r * Rc[c][r] */
    for (int c = 0; c < 3; ++c)
        for (int rr = 0; rr < 3; ++rr) M[c][rr] = s[rr] * Rc[c][rr];
    float dS[3][3] = {{dL_dcov3D[0], 0.5f * dL_dcov3D[1], 0.5f * dL_dcov3D[2]},
                      {0.5f * dL_dcov3D[1], dL_dcov3D[3], 0.5f * dL_dcov3D[4]},
                      {0.5f * dL_dcov3D[2], 0.5f * dL_dcov3D[4], dL_dcov3D[5]}};
    /* dL_dM = (2*M) * dSigma ; glm: (A*B)[c][r] = sum_k A[k][r]*B[c][k] */
    float dM[3][3];
    for (int c = 0; c < 3; ++c)
        for (int rr = 0; rr < 3; ++rr)
            dM[c][rr] = (2.0f * M[0][rr]) * dS[c][0] + (2.0f * M[1][rr]) * dS[c][1] + (2.0f * M[2][rr]) * dS[c][2];
    /* Rt = transpose(R): Rt[c][r] = Rc[r][c]; dMt[c][r] = dM[r][c] */
    float dMt[3][3];
    for (int c = 0; c < 3; ++c)
        for (int rr = 0; rr < 3; ++rr) dMt[c][rr] = dM[rr][c];
    for (int k = 0; k < 3; ++k)
        dL_dscale[k] = Rc[0][k] * dMt[k][0] + Rc[1][k] * dMt[k][1] + Rc[2][k] * dMt[k][2];
    for (int k = 0; k < 3; ++k)
        for (int rr = 0; rr < 3; ++rr) dMt[k][rr] *= s[k];
    dL_drot[0] = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
    dL_drot[1] = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) - 4 * x * (dMt[2][2] + dMt[1][1]);
    dL_drot[2] = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) - 4 * y * (dMt[2][2] + dMt[0][0]);
    dL_drot[3] = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) - 4 * z * (dMt[1][1] + dMt[0][0]);
}

/* dL/dcov3D from dL/dhat (6) through cov = M^T V M: the expanded sums of RAS/backward.cu:258-271
 * (same in VOX/backward.cu:157-170).  Mm[c*3+r]. Adds into dcov[6]. */
static void dcov3d_from_dhat(const float* Mm, const float* dh, float* dcov) {
#define M_(c, r) Mm[(c) * 3 + (r)]
    float da = dh[0], db = dh[1], dc = dh[2], dd = dh[3], de = dh[4], df = dh[5];
    dcov[0] += M_(0,0)*M_(0,0)*da + M_(0,0)*M_(1,0)*db + M_(0,0)*M_(2,0)*dc + M_(1,0)*M_(1,0)*dd + M_(1,0)*M_(2,0)*de + M_(2,0)*M_(2,0)*df;
    dcov[3] += M_(0,1)*M_(0,1)*da + M_(0,1)*M_(1,1)*db + M_(0,1)*M_(2,1)*dc + M_(1,1)*M_(1,1)*dd + M_(1,1)*M_(2,1)*de + M_(2,1)*M_(2,1)*df;
    dcov[5] += M_(0,2)*M_(0,2)*da + M_(0,2)*M_(1,2)*db + M_(0,2)*M_(2,2)*dc + M_(1,2)*M_(1,2)*dd + M_(1,2)*M_(2,2)*de + M_(2,2)*M_(2,2)*df;
    dcov[1] += 2*M_(0,0)*M_(0,1)*da + (M_(0,1)*M_(1,0)+M_(0,0)*M_(1,1))*db + (M_(0,1)*M_(2,0)+M_(0,0)*M_(2,1))*dc + 2*M_(1,0)*M_(1,1)*dd + (M_(1,1)*M_(2,0)+M_(1,0)*M_(2,1))*de + 2*M_(2,0)*M_(2,1)*df;
    dcov[2] += 2*M_(0,0)*M_(0,2)*da + (M_(0,2)*M_(1,0)+M_(0,0)*M_(1,2))*db + (M_(0,2)*M_(2,0)+M_(0,0)*M_(2,2))*dc + 2*M_(1,0)*M_(1,2)*dd + (M_(1,2)*M_(2,0)+M_(1,0)*M_(2,2))*de + 2*M_(2,0)*M_(2,2)*df;
    dcov[4] += 2*M_(0,1)*M_(0,2)*da + (M_(0,2)*M_(1,1)+M_(0,1)*M_(1,2))*db + (M_(0,2)*M_(2,1)+M_(0,1)*M_(2,2))*dc + 2*M_(1,1)*M_(1,2)*dd + (M_(1,2)*M_(2,1)+M_(1,1)*M_(2,2))*de + 2*M_(2,1)*M_(2,2)*df;
#undef M_
}

/* computeCov2DCUDA + preprocessCUDA backward, RAS/backward.cu:145-330 and :402-444.
 * Inputs: dL_dmean2D[3P], dL_dconic[4P], dL_dmu[P] from the render backward.
 * Outputs (zero-initialised here like the binding does, SUB/rasterize_points.cu:123-130):
 * dL_dmean3D[3P], dL_dcov3D[6P], dL_dscale[3P], dL_drot[4P]. */
void orc_raster_preprocess_backward(int P, const float* means, const int* radii, const float* scales,
                                    float scale_modifier, const float* rots, const float* cov3D /*6P*/,
                                    int have_scales, const float* view, const float* proj, int W, int H,
                                    float tan_fovx, float tan_fovy, int mode, const float* dL_dmean2D,
                                    const float* dL_dconic, const float* dL_dmu, float* dL_dmean3D,
                                    float* dL_dcov3D, float* dL_dscale, float* dL_drot) {
    const float h_y = H / (2.0f * tan_fovy), h_x = W / (2.0f * tan_fovx);
    memset(dL_dmean3D, 0, sizeof(float) * 3 * (size_t)P);
    memset(dL_dcov3D, 0, sizeof(float) * 6 * (size_t)P);
    memset(dL_dscale, 0, sizeof(float) * 3 * (size_t)P);
    memset(dL_drot, 0, sizeof(float) * 4 * (size_t)P);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; ++i) {
        if (!(radii[i] > 0)) continue;
        const float* c3 = cov3D + 6 * i;
        const float* mean = means + 3 * i;
        float dcx = dL_dconic[4 * i], dcy = dL_dconic[4 * i + 1], dcz = dL_dconic[4 * i + 3];
        float dmu = dL_dmu[i];
        float Mm[9], t[3], hat[6], txtz, tytz;
        raster_build_M(mean, view, h_x, h_y, tan_fovx, tan_fovy, mode, Mm, t, &txtz, &tytz);
        raster_cov_from_M(Mm, c3, hat);
        float x_grad_mul, y_grad_mul;
        if (mode == 0) {
            /* RAS/backward.cu:182-183 tests the already-clamped t, so both are always 1 */
            x_grad_mul = (t[0] < -1.3f || t[0] > 1.3f) ? 0.f : 1.f;
            y_grad_mul = (t[1] < -1.3f || t[1] > 1.3f) ? 0.f : 1.f;
        } else {
            float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
            x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
            y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
        }
        float a = hat[0], b = hat[1], c = hat[2], d = hat[3], e = hat[4], f = hat[5];
        float denom = a * d - b * b;
        float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        float diamond = denom;
        float circ = a * d * f + 2 * b * c * e - a * e * e - f * b * b - d * c * c;
        double musq = 2 * M_PI * circ / diamond;
        float muv = 0.f;
        if ((float)musq > 0.0f) muv = (float)sqrt(musq);
        float pi_mu = (float)(M_PI / (muv + 0.0000001f));
        float circ_diamond = circ / diamond;
        float dh[6] = {0, 0, 0, 0, 0, 0};
        float* dcov = dL_dcov3D + 6 * i;
        if (denom2inv != 0.0f && muv != 0.0f) {
            dh[0] = denom2inv * (-d * d * dcx + b * d * dcy + (denom - a * d) * dcz);
            dh[3] = denom2inv * (-a * a * dcz + a * b * dcy + (denom - a * d) * dcx);
            dh[1] = denom2inv * (2 * b * d * dcx - (denom + 2 * b * b) * dcy + 2 * a * b * dcz);
            dh[0] += pi_mu * ((d * f - e * e) / diamond - d * circ_diamond / diamond) * dmu;
            dh[1] += pi_mu * ((2 * c * e - 2 * f * b) / diamond + 2 * b * circ_diamond / diamond) * dmu;
            dh[2] += pi_mu * ((2 * b * e - 2 * d * c) / diamond) * dmu;
            dh[3] += pi_mu * ((a * f - c * c) / diamond - a * circ_diamond / diamond) * dmu;
            dh[4] += pi_mu * ((2 * b * c - 2 * a * e) / diamond) * dmu;
            dh[5] += pi_mu * ((a * d - b * b) / diamond) * dmu;
            dcov3d_from_dhat(Mm, dh, dcov);
        } else {
            for (int k = 0; k < 6; ++k) dcov[k] = 0.f;
        }
        float dmean[3] = {0.f, 0.f, 0.f};
        if (mode == 1) { /* RAS/backward.cu:279-329: dL/dM -> dL/dJ -> dL/dt -> dL/dmean (assign) */
#define M_(c, r) Mm[(c) * 3 + (r)]
            float va = c3[0], vb = c3[1], vc = c3[2], vd = c3[3], ve = c3[4], vf = c3[5];
            float m0a = M_(0,0)*va + M_(0,1)*vb + M_(0,2)*vc, m0b = M_(0,0)*vb + M_(0,1)*vd + M_(0,2)*ve, m0c = M_(0,0)*vc + M_(0,1)*ve + M_(0,2)*vf;
            float m1a = M_(1,0)*va + M_(1,1)*vb + M_(1,2)*vc, m1b = M_(1,0)*vb + M_(1,1)*vd + M_(1,2)*ve, m1c = M_(1,0)*vc + M_(1,1)*ve + M_(1,2)*vf;
            float m2a = M_(2,0)*va + M_(2,1)*vb + M_(2,2)*vc, m2b = M_(2,0)*vb + M_(2,1)*vd + M_(2,2)*ve, m2c = M_(2,0)*vc + M_(2,1)*ve + M_(2,2)*vf;
            float dM00 = 2*m0a*dh[0] + m1a*dh[1] + m2a*dh[2];
            float dM01 = 2*m0b*dh[0] + m1b*dh[1] + m2b*dh[2];
            float dM02 = 2*m0c*dh[0] + m1c*dh[1] + m2c*dh[2];
            float dM10 = m0a*dh[1] + 2*m1a*dh[3] + m2a*dh[4];
            float dM11 = m0b*dh[1] + 2*m1b*dh[3] + m2b*dh[4];
            float dM12 = m0c*dh[1] + 2*m1c*dh[3] + m2c*dh[4];
            float dM20 = m0a*dh[2] + m1a*dh[4] + 2*m2a*dh[5];
            float dM21 = m0b*dh[2] + m1b*dh[4] + 2*m2b*dh[5];
            float dM22 = m0c*dh[2] + m1c*dh[4] + 2*m2c*dh[5];
            /* W[k][r] = view[k+4r] */
#define W_(k, r) view[(k) + 4 * (r)]
            float dJ00 = W_(0,0)*dM00 + W_(0,1)*dM01 + W_(0,2)*dM02;
            float dJ02 = W_(2,0)*dM00 + W_(2,1)*dM01 + W_(2,2)*dM02;
            float dJ11 = W_(1,0)*dM10 + W_(1,1)*dM11 + W_(1,2)*dM12;
            float dJ12 = W_(2,0)*dM10 + W_(2,1)*dM11 + W_(2,2)*dM12;
            float dJ20 = W_(0,0)*dM20 + W_(0,1)*dM21 + W_(0,2)*dM22;
            float dJ21 = W_(1,0)*dM20 + W_(1,1)*dM21 + W_(1,2)*dM22;
            float dJ22 = W_(2,0)*dM20 + W_(2,1)*dM21 + W_(2,2)*dM22;
#undef W_
#undef M_
            float tx = t[0], ty = t[1], tz = t[2];
            float inv_tz = 1.f / tz, inv_tz2 = inv_tz * inv_tz, inv_tz3 = inv_tz2 * inv_tz;
            float cc = sqrtf(tx * tx + ty * ty + tz * tz);
            float icc3 = 1 / (cc * cc * cc);
            float dtx = x_grad_mul * (-h_x * inv_tz2 * dJ02 + (1 / cc - tx * tx * icc3) * dJ20 - tx * ty * icc3 * dJ21 - tx * tz * icc3 * dJ22);
            float dty = y_grad_mul * (-h_y * inv_tz2 * dJ12 - tx * ty * icc3 * dJ20 + (1 / cc - ty * ty * icc3) * dJ21 - ty * tz * icc3 * dJ22);
            float dtz = -h_x * inv_tz2 * dJ00 + 2 * h_x * tx * inv_tz3 * dJ02 - h_y * inv_tz2 * dJ11 + 2 * h_y * ty * inv_tz3 * dJ12 - tx * tz * icc3 * dJ20 - ty * tz * icc3 * dJ21 + (1 / cc - tz * tz * icc3) * dJ22;
            /* transformVec4x3Transpose, RAS/auxiliary.h:93-101 */
            dmean[0] = view[0] * dtx + view[1] * dty + view[2] * dtz;
            dmean[1] = view[4] * dtx + view[5] * dty + view[6] * dtz;
            dmean[2] = view[8] * dtx + view[9] * dty + view[10] * dtz;
        }
        /* preprocessCUDA backward, RAS/backward.cu:402-444 */
        float mx = mean[0], my = mean[1], mz = mean[2];
        float hw = proj[3] * mx + proj[7] * my + proj[11] * mz + proj[15];
        float m_w = 1.0f / (hw + 0.0000001f);
        float mul1 = (proj[0] * mx + proj[4] * my + proj[8] * mz + proj[12]) * m_w * m_w;
        float mul2 = (proj[1] * mx + proj[5] * my + proj[9] * mz + proj[13]) * m_w * m_w;
        float g2x = dL_dmean2D[3 * i], g2y = dL_dmean2D[3 * i + 1];
        dmean[0] += (proj[0] * m_w - proj[3] * mul1) * g2x + (proj[1] * m_w - proj[3] * mul2) * g2y;
        dmean[1] += (proj[4] * m_w - proj[7] * mul1) * g2x + (proj[5] * m_w - proj[7] * mul2) * g2y;
        dmean[2] += (proj[8] * m_w - proj[11] * mul1) * g2x + (proj[9] * m_w - proj[11] * mul2) * g2y;
        dL_dmean3D[3 * i] = dmean[0]; dL_dmean3D[3 * i + 1] = dmean[1]; dL_dmean3D[3 * i + 2] = dmean[2];
        if (have_scales) cov3d_backward(scales + 3 * i, scale_modifier, rots + 4 * i, dcov, dL_dscale + 3 * i, dL_drot + 4 * i);
    }
}

/* ----------------------------------------------------------------------------
 * Voxelizer forward
 * -------------------------------------------------------------------------- */

/* preprocessCUDA, VOX/forward.cu:58-178.  Outputs: radii_x/y/z[P], xyz_vol[3P], depth[P], cov3D[6P],
 * conic_opacity[7P], tiles_touched[P], cube[6P]=(x0,y0,z0,x1,y1,z1). Returns sum(tiles_touched). */
long long orc_voxel_preprocess(int P, const float* means, const float* scales, float scale_modifier,
                               const float* rots, const float* opac, const float* cov3D_precomp, int nx,
                               int ny, int nz, float sx, float sy, float sz, float cx, float cy, float cz,
                               int* radii_x, int* radii_y, int* radii_z, float* xyz_vol, float* depth,
                               float* cov3D, float* conic_opacity, uint32_t* tiles_touched, int* cube) {
    const int gx = (nx + VT - 1) / VT, gy = (ny + VT - 1) / VT, gz = (nz + VT - 1) / VT;
    const float fnx = (float)nx, fny = (float)ny, fnz = (float)nz;
    const float dvx = sx / fnx, dvy = sy / fny, dvz = sz / fnz;
    const float ix = 1.0f / dvx, iy = 1.0f / dvy, iz = 1.0f / dvz;
    long long total = 0;
#pragma omp parallel for reduction(+ : total) schedule(static)
    for (int i = 0; i < P; ++i) {
        radii_x[i] = radii_y[i] = radii_z[i] = 0;
        tiles_touched[i] = 0;
        depth[i] = 0.f;
        for (int k = 0; k < 3; ++k) xyz_vol[3 * i + k] = 0.f;
        for (int k = 0; k < 7; ++k) conic_opacity[7 * i + k] = 0.f;
        for (int k = 0; k < 6; ++k) cube[6 * i + k] = 0;
        const float* p = means + 3 * i;
        const float* c3;
        if (cov3D_precomp) {
            c3 = cov3D_precomp + 6 * i;
            if (cov3D) memcpy(cov3D + 6 * i, c3, 24);
        } else {
            cov3d_from_scale_rot(scales + 3 * i, scale_modifier, rots + 4 * i, cov3D + 6 * i);
            c3 = cov3D + 6 * i;
        }
        /* cov = D^T Vrk^T D with D = diag(1/dVoxel), VOX/forward.cu:110-118 */
        float a = (ix * c3[0]) * ix, b = (iy * c3[1]) * ix, c = (iz * c3[2]) * ix;
        float d = (iy * c3[3]) * iy, e = (iz * c3[4]) * iy, f = (iz * c3[5]) * iz;
        float ad = a * d, ae = a * e, bf = b * f, cd = c * d;
        float det = ad * f;
        det = fmaf((b + b) * c, e, det);
        det = fmaf(-e, ae, det);
        det = fmaf(-b, bf, det);
        det = fmaf(-c, cd, det);
        if (det == 0.0f) continue;
        float di = 1.0f / det;
        float inv_a = fmaf(d, f, -(e * e)) * di;
        float inv_b = fmaf(c, e, -bf) * di;
        float inv_c = fmaf(b, e, -cd) * di;
        float inv_d = fmaf(a, f, -(c * c)) * di;
        float inv_e = fmaf(b, c, -ae) * di;
        float inv_f = fmaf(-b, b, ad) * di;
        const float* s = scales + 3 * i; /* read unconditionally, VOX/forward.cu:137 */
        float ms3 = fmaxf(fmaxf(s[0], s[1]), s[2]) * 3.0f;
        float rx = ceilf(ms3 / dvx), ry = ceilf(ms3 / dvy), rz = ceilf(ms3 / dvz);
        float pvx = fmaf(sx, 0.5f, p[0] - cx) / dvx;
        float pvy = fmaf(sy, 0.5f, p[1] - cy) / dvy;
        float pvz = fmaf(sz, 0.5f, p[2] - cz) / dvz;
        if (pvx + rx < 0 || pvy + ry < 0 || pvz + rz < 0 || pvx - rx > fnx || pvy - ry > fny || pvz - rz > fnz) continue;
        /* getCube, VOX/auxiliary.h:27-39 */
        int x0 = imin(gx, imax(0, (int)((pvx - rx) * 0.125f)));
        int y0 = imin(gy, imax(0, (int)((pvy - ry) * 0.125f)));
        int z0 = imin(gz, imax(0, (int)((pvz - rz) * 0.125f)));
        int x1 = imin(gx, imax(0, (int)((((pvx + rx) + 8.0f) + -1.0f) * 0.125f)));
        int y1 = imin(gy, imax(0, (int)((((pvy + ry) + 8.0f) + -1.0f) * 0.125f)));
        int z1 = imin(gz, imax(0, (int)((((pvz + rz) + 8.0f) + -1.0f) * 0.125f)));
        int nt = (x1 - x0) * (y1 - y0) * (z1 - z0);
        if (nt == 0) continue;
        radii_x[i] = (int)rx; radii_y[i] = (int)ry; radii_z[i] = (int)rz;
        tiles_touched[i] = (uint32_t)nt;
        depth[i] = p[2];
        xyz_vol[3 * i] = pvx; xyz_vol[3 * i + 1] = pvy; xyz_vol[3 * i + 2] = pvz;
        float* co = conic_opacity + 7 * i;
        co[0] = inv_a; co[1] = inv_b; co[2] = inv_c; co[3] = inv_d; co[4] = inv_e; co[5] = inv_f; co[6] = opac[i];
        cube[6 * i] = x0; cube[6 * i + 1] = y0; cube[6 * i + 2] = z0;
        cube[6 * i + 3] = x1; cube[6 * i + 4] = y1; cube[6 * i + 5] = z1;
        total += nt;
    }
    return total;
}

/* power exactly as VOX/forward.cu:274 evaluates it: the 0.5 literal is a double, so the first term
 * is formed in float64 from a float32 sum and the whole expression stays in float64 until the
 * final float store. */
static inline float voxel_power(const float* co, float dx, float dy, float dz) {
    float s = co[0] * dx * dx + co[3] * dy * dy + co[5] * dz * dz;
    double pw = -0.5 * (double)s - (double)(co[1] * dx * dy) - (double)(co[2] * dx * dz) - (double)(co[4] * dy * dz);
    return (float)pw;
}

/* renderCUDA, VOX/forward.cu:183-315. out_volume index = x*ny*nz + y*nz + z. */
void orc_voxel_render(int nx, int ny, int nz, const uint32_t* ranges, const uint32_t* point_list,
                      const float* xyz_vol, const float* conic_opacity, float* out_volume, uint32_t* n_contrib) {
    const int gx = (nx + VT - 1) / VT, gy = (ny + VT - 1) / VT, gz = (nz + VT - 1) / VT;
#pragma omp parallel for schedule(dynamic, 1)
    for (int tile = 0; tile < gx * gy * gz; ++tile) {
        int tx = tile % gx, ty = (tile / gx) % gy, tz = tile / (gx * gy);
        uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        for (int lx = 0; lx < VT; ++lx)
            for (int ly = 0; ly < VT; ++ly)
                for (int lz = 0; lz < VT; ++lz) {
                    int vx = tx * VT + lx, vy = ty * VT + ly, vz = tz * VT + lz;
                    if (vx >= nx || vy >= ny || vz >= nz) continue;
                    float fx = (float)vx + 0.5f, fy = (float)vy + 0.5f, fz = (float)vz + 0.5f;
                    float C = 0.f;
                    uint32_t contributor = 0, last = 0;
                    for (uint32_t s = r0; s < r1; ++s) {
                        uint32_t g = point_list[s];
                        contributor++;
                        float dx = xyz_vol[3 * g] - fx, dy = xyz_vol[3 * g + 1] - fy, dz = xyz_vol[3 * g + 2] - fz;
                        const float* co = conic_opacity + 7 * g;
                        float power = voxel_power(co, dx, dy, dz);
                        if (power > 0.0f) continue;
                        float alpha = co[6] * expf(power);
                        if (alpha < 0.000001f) continue;
                        C += alpha;
                        last = contributor;
                    }
                    size_t vid = (size_t)nz * ny * vx + (size_t)nz * vy + vz;
                    out_volume[vid] = C;
                    if (n_contrib) n_contrib[vid] = last;
                }
    }
}

/* Voxelizer::forward, VOX/voxelizer_impl.cu:171-302. */
long long orc_voxel_forward(int P, const float* means, const float* scales, float scale_modifier,
                            const float* rots, const float* opac, const float* cov3D_precomp, int nx, int ny,
                            int nz, float sx, float sy, float sz, float cx, float cy, float cz,
                            float* out_volume, int* radii_x, int* radii_y, int* radii_z, float* xyz_vol,
                            float* depth, float* cov3D, float* conic_opacity, uint32_t* tiles_touched,
                            int* cube, uint32_t* n_contrib, uint64_t** keys_out, uint32_t** vals_out,
                            uint32_t** ranges_out) {
    const int gx = (nx + VT - 1) / VT, gy = (ny + VT - 1) / VT, gz = (nz + VT - 1) / VT;
    long long R = orc_voxel_preprocess(P, means, scales, scale_modifier, rots, opac, cov3D_precomp, nx, ny, nz,
                                       sx, sy, sz, cx, cy, cz, radii_x, radii_y, radii_z, xyz_vol, depth, cov3D,
                                       conic_opacity, tiles_touched, cube);
    uint64_t* keys = (uint64_t*)malloc((size_t)(R > 0 ? R : 1) * sizeof(uint64_t));
    uint32_t* vals = (uint32_t*)malloc((size_t)(R > 0 ? R : 1) * sizeof(uint32_t));
    uint32_t* ranges = (uint32_t*)malloc((size_t)gx * gy * gz * 2 * sizeof(uint32_t));
    orc_emit_keys(P, 3, cube, tiles_touched, depth, gx, gy, keys, vals);
    orc_sort_pairs((size_t)R, keys, vals);
    orc_tile_ranges((size_t)R, keys, gx * gy * gz, ranges);
    orc_voxel_render(nx, ny, nz, ranges, vals, xyz_vol, conic_opacity, out_volume, n_contrib);
    if (keys_out) *keys_out = keys; else free(keys);
    if (vals_out) *vals_out = vals; else free(vals);
    if (ranges_out) *ranges_out = ranges; else free(ranges);
    return R;
}

/* ----------------------------------------------------------------------------
 * Voxelizer backward
 * -------------------------------------------------------------------------- */

/* renderCUDA backward, VOX/backward.cu:216-374; float32 per-pair terms (float64 where the
 * reference's double literals promote them), float64 accumulation (see the rasterizer note).
 * dL_dmean3D_norm[3P] (already multiplied by dVoxel as the reference does), dL_dconic3D[6P], dL_dopacity[P]. */
void orc_voxel_render_backward(int P, int nx, int ny, int nz, float sx, float sy, float sz,
                               const uint32_t* ranges, const uint32_t* point_list, const float* xyz_vol,
                               const float* conic_opacity, const float* dL_dvol, float* dL_dmean3D_norm,
                               float* dL_dconic3D, float* dL_dopacity) {
    const int gx = (nx + VT - 1) / VT, gy = (ny + VT - 1) / VT, gz = (nz + VT - 1) / VT;
    const float dvx = sx / (float)nx, dvy = sy / (float)ny, dvz = sz / (float)nz;
    double* acc = (double*)calloc((size_t)P * 10, sizeof(double));
    for (int tile = 0; tile < gx * gy * gz; ++tile) {
        int tx = tile % gx, ty = (tile / gx) % gy, tz = tile / (gx * gy);
        uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        for (int lx = 0; lx < VT; ++lx)
            for (int ly = 0; ly < VT; ++ly)
                for (int lz = 0; lz < VT; ++lz) {
                    int vx = tx * VT + lx, vy = ty * VT + ly, vz = tz * VT + lz;
                    if (vx >= nx || vy >= ny || vz >= nz) continue;
                    float fx = (float)vx + 0.5f, fy = (float)vy + 0.5f, fz = (float)vz + 0.5f;
                    float dLp = dL_dvol[(size_t)nz * ny * vx + (size_t)nz * vy + vz];
                    for (uint32_t s = r0; s < r1; ++s) {
                        uint32_t g = point_list[s];
                        float dx = xyz_vol[3 * g] - fx, dy = xyz_vol[3 * g + 1] - fy, dz = xyz_vol[3 * g + 2] - fz;
                        const float* co = conic_opacity + 7 * g;
                        float power = voxel_power(co, dx, dy, dz);
                        if (power > 0.0f) continue;
                        float G = expf(power);
                        float alpha = co[6] * G;
                        if (alpha < 0.000001f) continue;
                        float dL_dalpha = dLp;
                        float dL_dG = co[6] * dL_dalpha;
                        float gdx = G * dx, gdy = G * dy, gdz = G * dz;
                        float dGx = -co[0] * gdx - co[1] * gdy - co[2] * gdz;
                        float dGy = -co[3] * gdy - co[1] * gdx - co[4] * gdz;
                        float dGz = -co[5] * gdz - co[2] * gdx - co[4] * gdy;
                        double* a = acc + (size_t)g * 10;
                        a[0] += (double)(dL_dG * dGx * dvx);
                        a[1] += (double)(dL_dG * dGy * dvy);
                        a[2] += (double)(dL_dG * dGz * dvz);
                        a[3] += (double)(float)(-0.5 * gdx * dx * dL_dG);
                        a[4] += (double)(float)(-1.0 * gdx * dy * dL_dG);
                        a[5] += (double)(float)(-1.0 * gdx * dz * dL_dG);
                        a[6] += (double)(float)(-0.5 * gdy * dy * dL_dG);
                        a[7] += (double)(float)(-1.0 * gdy * dz * dL_dG);
                        a[8] += (double)(float)(-0.5 * gdz * dz * dL_dG);
                        a[9] += (double)(G * dL_dalpha);
                    }
                }
    }
    for (int g = 0; g < P; ++g) {
        const double* a = acc + (size_t)g * 10;
        for (int k = 0; k < 3; ++k) dL_dmean3D_norm[3 * g + k] = (float)a[k];
        for (int k = 0; k < 6; ++k) dL_dconic3D[6 * g + k] = (float)a[3 + k];
        dL_dopacity[g] = (float)a[9];
    }
    free(acc);
}

/* computeCov3DCUDA + preprocessCUDA backward, VOX/backward.cu:86-213.
 * Outputs zero-initialised as SUB/voxelize_points.cu:111-117 does. */
void orc_voxel_preprocess_backward(int P, const int* radii_x, const int* radii_y, const int* radii_z,
                                   const float* scales, float scale_modifier, const float* rots,
                                   const float* cov3D, int have_scales, int nx, int ny, int nz, float sx,
                                   float sy, float sz, const float* dL_dmean3D_norm, const float* dL_dconic3D,
                                   float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot) {
    const float dvx = sx / (float)nx, dvy = sy / (float)ny, dvz = sz / (float)nz;
    const float ix = 1.0f / dvx, iy = 1.0f / dvy, iz = 1.0f / dvz;
    memset(dL_dmean3D, 0, sizeof(float) * 3 * (size_t)P);
    memset(dL_dcov3D, 0, sizeof(float) * 6 * (size_t)P);
    memset(dL_dscale, 0, sizeof(float) * 3 * (size_t)P);
    memset(dL_drot, 0, sizeof(float) * 4 * (size_t)P);
    const float Mm[9] = {ix, 0, 0, 0, iy, 0, 0, 0, iz};
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; ++i) {
        if (!(radii_x[i] > 0) || !(radii_y[i] > 0) || !(radii_z[i] > 0)) continue;
        const float* c3 = cov3D + 6 * i;
        const float* g = dL_dconic3D + 6 * i;
        float ga = g[0], gb = g[1], gc = g[2], gd = g[3], ge = g[4], gf = g[5];
        float a = (ix * c3[0]) * ix, b = (iy * c3[1]) * ix, c = (iz * c3[2]) * ix;
        float d = (iy * c3[3]) * iy, e = (iz * c3[4]) * iy, f = (iz * c3[5]) * iz;
        float denom = a * d * f + 2 * b * c * e - a * e * e - f * b * b - d * c * c;
        float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        float* dcov = dL_dcov3D + 6 * i;
        if (denom2inv != 0) {
            float n_da = d * f - e * e, n_db = 2 * c * e - 2 * f * b, n_dc = 2 * b * e - 2 * d * c;
            float n_dd = a * f - c * c, n_de = 2 * b * c - 2 * a * e, n_df = a * d - b * b;
            float ce_bf = c * e - b * f, be_cd = b * e - c * d, bc_ae = b * c - a * e;
            float dh[6];
            dh[0] = denom2inv * (-n_da*n_da*ga - ce_bf*n_da*gb - be_cd*n_da*gc + (f*denom-n_dd*n_da)*gd + (-e*denom-bc_ae*n_da)*ge + (d*denom-n_df*n_da)*gf);
            dh[1] = denom2inv * (-n_da*n_db*ga + (-f*denom-ce_bf*n_db)*gb + (e*denom-be_cd*n_db)*gc - n_dd*n_db*gd + (c*denom-bc_ae*n_db)*ge + (-2*b*denom-n_df*n_db)*gf);
            dh[2] = denom2inv * (-n_da*n_dc*ga + (e*denom-ce_bf*n_dc)*gb + (-d*denom-be_cd*n_dc)*gc + (-2*c*denom-n_dd*n_dc)*gd + (b*denom-bc_ae*n_dc)*ge - n_df*n_dc*gf);
            dh[3] = denom2inv * ((f*denom-n_da*n_dd)*ga - ce_bf*n_dd*gb + (-c*denom-be_cd*n_dd)*gc - n_dd*n_dd*gd - bc_ae*n_dd*ge + (a*denom-n_df*n_dd)*gf);
            dh[4] = denom2inv * ((-2*e*denom-n_da*n_de)*ga + (c*denom-ce_bf*n_de)*gb + (b*denom-be_cd*n_de)*gc - n_dd*n_de*gd + (-a*denom-bc_ae*n_de)*ge + -n_df*n_de*gf);
            dh[5] = denom2inv * ((d*denom-n_da*n_df)*ga + (-b*denom-ce_bf*n_df)*gb - be_cd*n_df*gc + (a*denom-n_dd*n_df)*gd - bc_ae*n_df*ge - n_df*n_df*gf);
            dcov3d_from_dhat(Mm, dh, dcov);
        } else {
            for (int k = 0; k < 6; ++k) dcov[k] = 0.f;
        }
        for (int k = 0; k < 3; ++k) dL_dmean3D[3 * i + k] = dL_dmean3D_norm[3 * i + k];
        if (have_scales) cov3d_backward(scales + 3 * i, scale_modifier, rots + 4 * i, dcov, dL_dscale + 3 * i, dL_drot + 4 * i);
    }
}

/* checkFrustum / markVisible, RAS/rasterizer_impl.cu:54-66, :141-153 */
void orc_mark_visible(int P, const float* means, const float* view, const float* proj, unsigned char* present) {
    (void)proj;
    for (int i = 0; i < P; ++i) {
        const float* p = means + 3 * i;
        present[i] = xform_row(view, 2, p[0], p[1], p[2]) > 0.2f;
    }
}

/* simple_knn._C.distCUDA2 (called at r2_gaussian/gaussian/gaussian_model.py:144-150).  The upstream extension
 * (gitlab.inria.fr/bkerbl/simple-knn) is an un-vendored submodule of the reference, so this restates its
 * published result -- for every point the mean of the three smallest squared distances to OTHER points, kept
 * in ascending order from FLT_MAX placeholders (updateKBest<3>) -- by brute force.  PARITY UNPINNED against
 * the upstream binary (absent); pinned against an independent float64 k-d tree in tests/test_oracle_cpu.py. */
static float knn3_one(int P, const float* pts, int i) {
    float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    for (int j = 0; j < P; ++j) {
        if (j == i) continue;
        const float dx = x - pts[3 * (size_t)j], dy = y - pts[3 * (size_t)j + 1], dz = z - pts[3 * (size_t)j + 2];
        const float d = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
        if (d < b2) {
            if (d < b1) {
                b2 = b1;
                if (d < b0) { b1 = b0; b0 = d; }
                else b1 = d;
            } else b2 = d;
        }
    }
    return ((b0 + b1) + b2) / 3.0f;
}

/* orc_knn3_mean_dist2's result for the n_query points idx[0 .. n_query-1] only (out[k] belongs to point idx[k]): the
 * same loop over all P points, so a cloud of millions can be checked at chosen points in O(n_query * P). */
void orc_knn3_mean_dist2_at(int P, const float* pts, int n_query, const int* idx, float* out) {
#pragma omp parallel for schedule(dynamic, 16)
    for (int k = 0; k < n_query; ++k) out[k] = knn3_one(P, pts, idx[k]);
}

void orc_knn3_mean_dist2(int P, const float* pts, float* out) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; ++i) out[i] = knn3_one(P, pts, i);
}

int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

void orc_set_num_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}
