// r2x_scene.cu -- depth-tested rasterization of triangles and line segments (the scene view: meshes, boxes, camera
// glyphs with textured image planes).  include/r2x.h states the model.
//
// Three passes on one stream, every frame of a call on gridDim.z (or in the records), so an orbit is one call:
//   setup   one thread per (primitive, frame): clip, project, snap, bound.  A primitive whose clamped pixel box is at
//           most R2X_SV_TILE pixels on each side is rasterized by that thread; a larger one appends a record (box,
//           tiles) to the scratch list.
//   scan    one CTA: exclusive scan of the records' tile counts (their order is the order of the atomic appends, which
//           changes nothing: every covered pixel is an atomicMin, so the result does not depend on who writes first).
//   tiles   a grid-stride loop over every tile of every record, one CTA of 16 x 16 threads per tile, one pixel each.
//   resolve one thread per pixel: background, or the winning primitive shaded.
// Projection, snapping, the line distance and the depth are float64 with explicit round-to-nearest operations, and the
// edge functions are int64, so a plain float64 / integer statement of the model (tests/scene_view_oracle.py) gives the
// same coverage and depth bits.
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {
namespace {

constexpr int SV_TILE = R2X_SV_TILE;
constexpr int SV_THREADS = SV_TILE * SV_TILE;
constexpr int SV_MAX_GRID = 65535;
constexpr int SV_MAX_POLY = 8;                    // a triangle clipped by 5 planes
constexpr int SV_SCAN_THREADS = 1024;
constexpr int SV_TILE_CTAS = 4096;
constexpr unsigned long long SV_EMPTY = ~0ull;
constexpr double SV_SUB = 256.0;                  // fixed point: 1/256 pixel

struct SvParams {
    int n_prims, n_frames, H, W, parallel, n_tex, th, tw, K;
    double near;
    float bg[3];
};

struct SvRecord {
    int prim, frame, x0, y0, x1, y1, tx, ty;
    long long base;
};

struct SvCounters {
    unsigned int n_records;
    unsigned int pad;
    unsigned long long tiles;
};

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

struct Cam {
    double P[3], f[3], r[3], u[3], p;
};

__device__ __forceinline__ Cam load_cam(const float* __restrict__ cameras, int frame) {
    const float* c = cameras + (size_t)frame * R2X_SV_CAMERA_FLOATS;
    Cam k;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        k.P[i] = __ldg(c + i);
        k.f[i] = __ldg(c + 3 + i);
        k.r[i] = __ldg(c + 6 + i);
        k.u[i] = __ldg(c + 9 + i);
    }
    k.p = __ldg(c + 12);
    return k;
}

__device__ __forceinline__ double dot3(const double* a, const double* b) {
    return dadd(dadd(dmul(a[0], b[0]), dmul(a[1], b[1])), dmul(a[2], b[2]));
}

// world point -> camera coordinates (x right, y up, z along the view direction)
__device__ __forceinline__ void to_cam(const Cam& k, const double* __restrict__ X, double* c) {
    const double d[3] = {dsub(__ldg(X), k.P[0]), dsub(__ldg(X + 1), k.P[1]), dsub(__ldg(X + 2), k.P[2])};
    c[0] = dot3(d, k.r);
    c[1] = dot3(d, k.u);
    c[2] = dot3(d, k.f);
}

// signed distance of a camera-space point to clip plane j (inside iff >= 0): 0 near, 1-4 the guard band
__device__ __forceinline__ double plane(const SvParams& q, const Cam& k, int j, const double* c) {
    if (j == 0) return dsub(c[2], q.near);
    const double g = q.parallel ? dmul(R2X_SV_GUARD, k.p) : dmul(dmul(R2X_SV_GUARD, k.p), c[2]);
    const double s = (j == 1 || j == 3) ? c[(j - 1) >> 1] : -c[(j - 1) >> 1];
    return dsub(g, s);
}

// the point where the edge from the inside point a (da >= 0) to the outside point b (db < 0) meets the plane
__device__ __forceinline__ void cut(const double* a, const double* b, double da, double db, double* o) {
    const double t = ddiv(da, dsub(da, db));
#pragma unroll
    for (int i = 0; i < 3; ++i) o[i] = dadd(a[i], dmul(t, dsub(b[i], a[i])));
}

__device__ __forceinline__ void project(const SvParams& q, const Cam& k, const double* c, double& sx, double& sy) {
    const double den = q.parallel ? k.p : dmul(c[2], k.p);
    sx = dadd(0.5 * q.W, ddiv(c[0], den));
    sy = dsub(0.5 * q.H, ddiv(c[1], den));
}

__device__ __forceinline__ long long snap(double s) { return __double2ll_rn(dmul(s, SV_SUB)); }

// the pixel-centre offsets of the volume renderer: a = ((x + 1/2) - W/2) p, b = ((H/2 - y) - 1/2) p
__device__ __forceinline__ void pixel_ab(const SvParams& q, const Cam& k, int x, int y, double& a, double& b) {
    a = dmul(((double)x + 0.5) - 0.5 * q.W, k.p);
    b = dmul((0.5 * q.H - (double)y) - 0.5, k.p);
}

__device__ __forceinline__ float depth_key_f(const SvParams& q, double z) {
    return __double2float_rn(z >= q.near ? z : q.near);   // NaN -> near
}

// an ellipsoid: centre, rotation (columns: the axes), semi-axes and their inverses
struct Ell {
    double c[3], R[3][3], s[3], k[3];
};

__device__ void load_ell(const double* __restrict__ pos, const float* __restrict__ attr, int id, Ell& E) {
    const double* X = pos + (size_t)id * 9;
    const float* at = attr + (size_t)id * R2X_SV_ATTR;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        E.c[i] = __ldg(X + i);
        E.s[i] = __ldg(X + 3 + i);
        E.k[i] = ddiv(1.0, E.s[i]);
    }
    double w = __ldg(at + 3), x = __ldg(at + 4), y = __ldg(at + 5), z = __ldg(at + 6);
    const double m = __dsqrt_rn(dadd(dadd(dadd(dmul(w, w), dmul(x, x)), dmul(y, y)), dmul(z, z)));
    w = ddiv(w, m); x = ddiv(x, m); y = ddiv(y, m); z = ddiv(z, m);
    E.R[0][0] = dsub(1.0, dmul(2.0, dadd(dmul(y, y), dmul(z, z))));
    E.R[0][1] = dmul(2.0, dsub(dmul(x, y), dmul(w, z)));
    E.R[0][2] = dmul(2.0, dadd(dmul(x, z), dmul(w, y)));
    E.R[1][0] = dmul(2.0, dadd(dmul(x, y), dmul(w, z)));
    E.R[1][1] = dsub(1.0, dmul(2.0, dadd(dmul(x, x), dmul(z, z))));
    E.R[1][2] = dmul(2.0, dsub(dmul(y, z), dmul(w, x)));
    E.R[2][0] = dmul(2.0, dsub(dmul(x, z), dmul(w, y)));
    E.R[2][1] = dmul(2.0, dadd(dmul(y, z), dmul(w, x)));
    E.R[2][2] = dsub(1.0, dmul(2.0, dadd(dmul(x, x), dmul(y, y))));
}

// o = diag(k) R^T v: v in the ellipsoid's unit-sphere frame
__device__ __forceinline__ void ell_local(const Ell& E, const double* v, double* o) {
#pragma unroll
    for (int j = 0; j < 3; ++j)
        o[j] = dmul(dadd(dadd(dmul(E.R[0][j], v[0]), dmul(E.R[1][j], v[1])), dmul(E.R[2][j], v[2])), E.k[j]);
}

// the ray O + t D of pixel (x, y); t is the camera depth
__device__ __forceinline__ void pixel_ray(const SvParams& q, const Cam& k, int x, int y, double* O, double* D) {
    double a, b;
    pixel_ab(q, k, x, y, a, b);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (q.parallel) {
            O[i] = dadd(dadd(k.P[i], dmul(a, k.r[i])), dmul(b, k.u[i]));
            D[i] = k.f[i];
        } else {
            O[i] = k.P[i];
            D[i] = dadd(dadd(k.f[i], dmul(a, k.r[i])), dmul(b, k.u[i]));
        }
    }
}

// whether the ray hits the ellipsoid at a depth >= near, and the depth of the visible surface
__device__ __forceinline__ bool ell_hit(const SvParams& q, const Ell& E, const double* O, const double* D, double& z) {
    const double w[3] = {dsub(O[0], E.c[0]), dsub(O[1], E.c[1]), dsub(O[2], E.c[2])};
    double e[3], g[3];
    ell_local(E, w, e);
    ell_local(E, D, g);
    const double A = dot3(g, g), B = dot3(g, e), C = dsub(dot3(e, e), 1.0);
    const double disc = dsub(dmul(B, B), dmul(A, C));
    if (!(disc >= 0.0)) return false;
    const double h = -dadd(B, copysign(__dsqrt_rn(disc), B));   // no cancellation
    const double t1 = ddiv(h, A), t2 = h != 0.0 ? ddiv(C, h) : t1;
    const double lo = fmin(t1, t2), hi = fmax(t1, t2);
    if (!(hi >= q.near)) return false;
    z = lo >= q.near ? lo : hi;
    return true;
}

// the image-plane range (b1 -+ d) / a2 of the two tangent planes through the camera along one screen axis
__device__ __forceinline__ void tangent_range(double cx, double cz, double sxz, double sxx, double a2, double& lo,
                                              double& hi) {
    const double b1 = dsub(dmul(cx, cz), sxz), c0 = dsub(dmul(cx, cx), sxx);
    const double d = __dsqrt_rn(fmax(dsub(dmul(b1, b1), dmul(a2, c0)), 0.0));
    lo = ddiv(dsub(b1, d), a2);
    hi = ddiv(dadd(b1, d), a2);
}

// a primitive in one frame, ready for the pixel test
struct Geom {
    bool line, ell;
    Ell E;                           // ellipsoid
    int nv;                          // triangle: clipped polygon size (0: nothing left); line: 2 or 0
    long long X[SV_MAX_POLY], Y[SV_MAX_POLY];
    double V[3][3];                  // triangle: camera-space vertices (unclipped), for the plane
    double n[3], c;                  // triangle plane n . X = c in camera space
    double ax, ay, bx, by, za, zb, r; // line: snapped end points in pixels, their camera depths, half width
    int x0, y0, x1, y1;              // clamped pixel box (x0 > x1 or y0 > y1: empty)
};

__device__ __forceinline__ long long floor256(long long v) { return v >> 8; }   // floor(v / 256)

__device__ void build_geom(const SvParams& q, const Cam& k, const double* __restrict__ pos, const int* __restrict__ meta,
                           const float* __restrict__ attr, int id, Geom& g) {
    const double* X = pos + (size_t)id * 9;
    const int kind = __ldg(meta + 2 * (size_t)id);
    g.line = kind == R2X_SV_LINE;
    g.ell = kind == R2X_SV_ELLIPSOID;
    g.x0 = 0; g.y0 = 0; g.x1 = -1; g.y1 = -1;
    if (g.ell) {
        g.nv = 0;
        load_ell(pos, attr, id, g.E);
        double cc[3], M[3][3];
        to_cam(k, X, cc);
        const double* rows[3] = {k.r, k.u, k.f};
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j)
                M[i][j] = dmul(dadd(dadd(dmul(rows[i][0], g.E.R[0][j]), dmul(rows[i][1], g.E.R[1][j])),
                                    dmul(rows[i][2], g.E.R[2][j])), g.E.s[j]);
        double S[3][3];   // Sigma in camera coordinates
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b)
                S[a][b] = dadd(dadd(dmul(M[a][0], M[b][0]), dmul(M[a][1], M[b][1])), dmul(M[a][2], M[b][2]));
        const double sz = __dsqrt_rn(S[2][2]);
        if (dadd(cc[2], sz) < q.near) return;
        g.nv = 1;
        double lx, hx, ly, hy;
        if (q.parallel) {
            const double sx = __dsqrt_rn(S[0][0]), sy = __dsqrt_rn(S[1][1]);
            lx = dadd(0.5 * q.W, ddiv(dsub(cc[0], sx), k.p));
            hx = dadd(0.5 * q.W, ddiv(dadd(cc[0], sx), k.p));
            ly = dsub(0.5 * q.H, ddiv(dadd(cc[1], sy), k.p));
            hy = dsub(0.5 * q.H, ddiv(dsub(cc[1], sy), k.p));
        } else {
            const double a2 = dsub(dmul(cc[2], cc[2]), S[2][2]);
            if (!(dsub(cc[2], sz) >= q.near) || !(a2 > 0.0)) {   // the camera is inside or near it: every pixel
                g.x0 = 0; g.y0 = 0; g.x1 = q.W - 1; g.y1 = q.H - 1;
                return;
            }
            double lo, hi;
            tangent_range(cc[0], cc[2], S[0][2], S[0][0], a2, lo, hi);
            lx = dadd(0.5 * q.W, ddiv(lo, k.p));
            hx = dadd(0.5 * q.W, ddiv(hi, k.p));
            tangent_range(cc[1], cc[2], S[1][2], S[1][1], a2, lo, hi);
            ly = dsub(0.5 * q.H, ddiv(hi, k.p));
            hy = dsub(0.5 * q.H, ddiv(lo, k.p));
        }
        g.x0 = (int)fmin(fmax(dsub(floor(lx), 1.0), 0.0), (double)q.W);
        g.x1 = (int)fmax(fmin(dadd(floor(hx), 1.0), (double)(q.W - 1)), -1.0);
        g.y0 = (int)fmin(fmax(dsub(floor(ly), 1.0), 0.0), (double)q.H);
        g.y1 = (int)fmax(fmin(dadd(floor(hy), 1.0), (double)(q.H - 1)), -1.0);
        return;
    }
    if (g.line) {
        double a[3], b[3];
        to_cam(k, X, a);
        to_cam(k, X + 3, b);
        g.nv = 0;
        for (int j = 0; j < 5; ++j) {
            const double da = plane(q, k, j, a), db = plane(q, k, j, b);
            if (da < 0.0 && db < 0.0) return;
            if (da < 0.0) {
                double o[3];
                cut(b, a, db, da, o);
                a[0] = o[0]; a[1] = o[1]; a[2] = o[2];
            } else if (db < 0.0) {
                double o[3];
                cut(a, b, da, db, o);
                b[0] = o[0]; b[1] = o[1]; b[2] = o[2];
            }
        }
        double sx, sy;
        project(q, k, a, sx, sy);
        g.ax = (double)snap(sx) / SV_SUB;
        g.ay = (double)snap(sy) / SV_SUB;
        project(q, k, b, sx, sy);
        g.bx = (double)snap(sx) / SV_SUB;
        g.by = (double)snap(sy) / SV_SUB;
        g.za = a[2];
        g.zb = b[2];
        g.r = 0.5 * (double)__ldg(attr + (size_t)id * R2X_SV_ATTR + 3);
        g.nv = 2;
        const double lx = dsub(dsub(fmin(g.ax, g.bx), g.r), 0.5), hx = dsub(dadd(fmax(g.ax, g.bx), g.r), 0.5);
        const double ly = dsub(dsub(fmin(g.ay, g.by), g.r), 0.5), hy = dsub(dadd(fmax(g.ay, g.by), g.r), 0.5);
        g.x0 = (int)fmax(ceil(lx), 0.0);
        g.x1 = (int)fmin(floor(hx), (double)(q.W - 1));
        g.y0 = (int)fmax(ceil(ly), 0.0);
        g.y1 = (int)fmin(floor(hy), (double)(q.H - 1));
        return;
    }
    // triangle: Sutherland-Hodgman against the 5 planes; every cut is formed from the edge's inside end to its outside
    // end, so two triangles sharing an edge get the same cut points
    double poly[SV_MAX_POLY][3], tmp[SV_MAX_POLY][3];
    for (int v = 0; v < 3; ++v) {
        to_cam(k, X + 3 * v, g.V[v]);
        poly[v][0] = g.V[v][0]; poly[v][1] = g.V[v][1]; poly[v][2] = g.V[v][2];
    }
    int n = 3;
    for (int j = 0; j < 5 && n > 0; ++j) {
        int m = 0;
        for (int v = 0; v < n; ++v) {
            const double* a = poly[v];
            const double* b = poly[(v + 1) % n];
            const double da = plane(q, k, j, a), db = plane(q, k, j, b);
            if (da >= 0.0) {
                tmp[m][0] = a[0]; tmp[m][1] = a[1]; tmp[m][2] = a[2];
                ++m;
            }
            if ((da >= 0.0) != (db >= 0.0)) {
                if (da >= 0.0) cut(a, b, da, db, tmp[m]);
                else cut(b, a, db, da, tmp[m]);
                ++m;
            }
        }
        n = m;
        for (int v = 0; v < n; ++v) {
            poly[v][0] = tmp[v][0]; poly[v][1] = tmp[v][1]; poly[v][2] = tmp[v][2];
        }
    }
    g.nv = n;
    if (n < 3) {
        g.nv = 0;
        return;
    }
    long long lx = LLONG_MAX, ly = LLONG_MAX, hx = LLONG_MIN, hy = LLONG_MIN;
    for (int v = 0; v < n; ++v) {
        double sx, sy;
        project(q, k, poly[v], sx, sy);
        g.X[v] = snap(sx);
        g.Y[v] = snap(sy);
        lx = min(lx, g.X[v]); hx = max(hx, g.X[v]);
        ly = min(ly, g.Y[v]); hy = max(hy, g.Y[v]);
    }
    // pixel x is a candidate iff lx <= 256 x + 128 <= hx
    g.x0 = (int)max(floor256(lx - 128 + 255), 0ll);
    g.x1 = (int)min(floor256(hx - 128), (long long)q.W - 1);
    g.y0 = (int)max(floor256(ly - 128 + 255), 0ll);
    g.y1 = (int)min(floor256(hy - 128), (long long)q.H - 1);
    double e1[3], e2[3];
    for (int i = 0; i < 3; ++i) {
        e1[i] = dsub(g.V[1][i], g.V[0][i]);
        e2[i] = dsub(g.V[2][i], g.V[0][i]);
    }
    g.n[0] = dsub(dmul(e1[1], e2[2]), dmul(e1[2], e2[1]));
    g.n[1] = dsub(dmul(e1[2], e2[0]), dmul(e1[0], e2[2]));
    g.n[2] = dsub(dmul(e1[0], e2[1]), dmul(e1[1], e2[0]));
    g.c = dot3(g.n, g.V[0]);
}

// edge (a -> b) owns the pixel centres on it iff it is a top or left edge of a triangle of positive area
__device__ __forceinline__ bool edge_in(long long ax, long long ay, long long bx, long long by, long long px,
                                        long long py) {
    const long long dx = bx - ax, dy = by - ay;
    const long long e = dx * (py - ay) - dy * (px - ax);
    return e > 0 || (e == 0 && (dy < 0 || (dy == 0 && dx > 0)));
}

// the depth at pixel (x, y) of the triangle plane: z = c / (n . (a, b, 1)) or (c - n_x a - n_y b) / n_z
__device__ __forceinline__ double tri_depth(const SvParams& q, const Geom& g, double a, double b) {
    if (q.parallel) return ddiv(dsub(dsub(g.c, dmul(g.n[0], a)), dmul(g.n[1], b)), g.n[2]);
    return ddiv(g.c, dadd(dadd(dmul(g.n[0], a), dmul(g.n[1], b)), g.n[2]));
}

// whether (x, y) is covered, and its depth
__device__ __forceinline__ bool cover(const SvParams& q, const Cam& k, const Geom& g, int x, int y, double& z) {
    double a, b;
    if (g.ell) {
        double O[3], D[3];
        pixel_ray(q, k, x, y, O, D);
        return ell_hit(q, g.E, O, D, z);
    }
    if (g.line) {
        const double cx = (double)x + 0.5, cy = (double)y + 0.5;
        const double dx = dsub(g.bx, g.ax), dy = dsub(g.by, g.ay), ex = dsub(cx, g.ax), ey = dsub(cy, g.ay);
        const double len2 = dadd(dmul(dx, dx), dmul(dy, dy));
        double t = 0.0;
        if (len2 > 0.0) t = fmin(fmax(ddiv(dadd(dmul(ex, dx), dmul(ey, dy)), len2), 0.0), 1.0);
        const double qx = dsub(ex, dmul(t, dx)), qy = dsub(ey, dmul(t, dy));
        if (!(dadd(dmul(qx, qx), dmul(qy, qy)) <= dmul(g.r, g.r))) return false;
        if (q.parallel) z = dadd(g.za, dmul(t, dsub(g.zb, g.za)));
        else z = ddiv(1.0, dadd(ddiv(dsub(1.0, t), g.za), ddiv(t, g.zb)));
        return true;
    }
    const long long px = 256ll * x + 128, py = 256ll * y + 128;
    bool in = false;
    for (int v = 1; v + 1 < g.nv && !in; ++v) {
        long long bx = g.X[v], by = g.Y[v], cx = g.X[v + 1], cy = g.Y[v + 1];
        const long long ax = g.X[0], ay = g.Y[0];
        const long long area = (bx - ax) * (cy - ay) - (by - ay) * (cx - ax);
        if (area == 0) continue;
        if (area < 0) {
            long long t = bx; bx = cx; cx = t;
            t = by; by = cy; cy = t;
        }
        in = edge_in(ax, ay, bx, by, px, py) && edge_in(bx, by, cx, cy, px, py) && edge_in(cx, cy, ax, ay, px, py);
    }
    if (!in) return false;
    pixel_ab(q, k, x, y, a, b);
    z = tri_depth(q, g, a, b);
    return true;
}

__device__ __forceinline__ void write_key(const SvParams& q, unsigned long long* keys, int frame, int x, int y,
                                          double z, int id) {
    const unsigned long long key = ((unsigned long long)__float_as_uint(depth_key_f(q, z)) << 32) | (unsigned)id;
    atomicMin(keys + ((long long)frame * q.H + y) * q.W + x, key);
}

__global__ void __launch_bounds__(256) sv_setup_kernel(SvParams q, const double* __restrict__ pos,
                                                       const int* __restrict__ meta, const float* __restrict__ attr,
                                                       const float* __restrict__ cameras, unsigned long long* keys,
                                                       SvCounters* cnt, SvRecord* rec) {
    const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= q.n_prims) return;
    const int frame = blockIdx.z;
    const Cam k = load_cam(cameras, frame);
    Geom g;
    build_geom(q, k, pos, meta, attr, (int)id, g);
    if (g.nv == 0 || g.x0 > g.x1 || g.y0 > g.y1) return;
    if (g.x1 - g.x0 < SV_TILE && g.y1 - g.y0 < SV_TILE) {
        for (int y = g.y0; y <= g.y1; ++y)
            for (int x = g.x0; x <= g.x1; ++x) {
                double z;
                if (cover(q, k, g, x, y, z)) write_key(q, keys, frame, x, y, z, (int)id);
            }
        return;
    }
    const unsigned r = atomicAdd(&cnt->n_records, 1u);
    SvRecord o;
    o.prim = (int)id; o.frame = frame; o.x0 = g.x0; o.y0 = g.y0; o.x1 = g.x1; o.y1 = g.y1;
    o.tx = (g.x1 - g.x0) / SV_TILE + 1;
    o.ty = (g.y1 - g.y0) / SV_TILE + 1;
    o.base = 0;
    rec[r] = o;
}

__global__ void __launch_bounds__(SV_SCAN_THREADS) sv_scan_kernel(SvCounters* cnt, SvRecord* rec) {
    __shared__ long long s_warp[SV_SCAN_THREADS / 32];
    __shared__ long long s_run;
    const int n = (int)cnt->n_records, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_run = 0;
    __syncthreads();
    for (int start = 0; start < n; start += SV_SCAN_THREADS) {
        const int i = start + threadIdx.x;
        const long long v = i < n ? (long long)rec[i].tx * rec[i].ty : 0;
        long long incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            long long w = s_warp[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long t = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += t;
            }
            s_warp[lane] = w;   // inclusive over warps
        }
        __syncthreads();
        const long long before = s_run + (warp ? s_warp[warp - 1] : 0) + incl - v;
        if (i < n) rec[i].base = before;
        __syncthreads();
        if (threadIdx.x == SV_SCAN_THREADS - 1) s_run = before + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) cnt->tiles = (unsigned long long)s_run;
}

__global__ void __launch_bounds__(SV_THREADS) sv_tile_kernel(SvParams q, const double* __restrict__ pos,
                                                             const int* __restrict__ meta,
                                                             const float* __restrict__ attr,
                                                             const float* __restrict__ cameras, unsigned long long* keys,
                                                             const SvCounters* cnt, const SvRecord* rec) {
    const long long total = (long long)cnt->tiles;
    const int nrec = (int)cnt->n_records;
    for (long long t = blockIdx.x; t < total; t += gridDim.x) {
        int lo = 0, hi = nrec - 1;   // the last record whose base <= t
        while (lo < hi) {
            const int mid = lo + ((hi - lo + 1) >> 1);   // lo + hi + 1 passes INT_MAX past 2^30 records
            if (rec[mid].base <= t) lo = mid;
            else hi = mid - 1;
        }
        const SvRecord r = rec[lo];
        const long long local = t - r.base;
        const int x = r.x0 + (int)(local % r.tx) * SV_TILE + (int)threadIdx.x;
        const int y = r.y0 + (int)(local / r.tx) * SV_TILE + (int)threadIdx.y;
        if (x > r.x1 || y > r.y1) continue;
        const Cam k = load_cam(cameras, r.frame);
        Geom g;
        build_geom(q, k, pos, meta, attr, r.prim, g);
        double z;
        if (cover(q, k, g, x, y, z)) write_key(q, keys, r.frame, x, y, z, r.prim);
    }
}

// the two-sided headlight shade A + (1 - A) min(|N.D| / sqrt(N.N D.D), 1) of normal N along the ray D (A if N = 0)
__device__ __forceinline__ double headlight(const double* N, const double* D) {
    const double nn = dot3(N, N), dd = dot3(D, D);
    double lam = 0.0;
    if (nn > 0.0) lam = fmin(fabs(ddiv(dot3(N, D), __dsqrt_rn(dmul(nn, dd)))), 1.0);
    return dadd(R2X_SV_AMBIENT, dmul(1.0 - R2X_SV_AMBIENT, lam));
}

__device__ __forceinline__ float fblend(float a, float b, float w) {
    return __fadd_rn(__fmul_rn(__fsub_rn(1.0f, w), a), __fmul_rn(w, b));
}

__global__ void __launch_bounds__(SV_THREADS) sv_resolve_kernel(SvParams q, const double* __restrict__ pos,
                                                                const int* __restrict__ meta,
                                                                const float* __restrict__ attr,
                                                                const float* __restrict__ tex,
                                                                const float* __restrict__ lut,
                                                                const float* __restrict__ cameras,
                                                                const unsigned long long* __restrict__ keys,
                                                                float* __restrict__ rgb) {
    const int x = blockIdx.x * SV_TILE + threadIdx.x, y = blockIdx.y * SV_TILE + threadIdx.y, frame = blockIdx.z;
    if (x >= q.W || y >= q.H) return;
    const long long px = ((long long)frame * q.H + y) * q.W + x;
    const unsigned long long key = keys[px];
    float out[3] = {q.bg[0], q.bg[1], q.bg[2]};
    if (key != SV_EMPTY) {
        const int id = (int)(unsigned)(key & 0xffffffffu);
        const int kind = __ldg(meta + 2 * (size_t)id);
        const float* at = attr + (size_t)id * R2X_SV_ATTR;
        if (kind == R2X_SV_LINE || kind == R2X_SV_FLAT) {
            out[0] = __ldg(at); out[1] = __ldg(at + 1); out[2] = __ldg(at + 2);
        } else if (kind == R2X_SV_ELLIPSOID) {
            const Cam k = load_cam(cameras, frame);
            Ell E;
            load_ell(pos, attr, id, E);
            double O[3], D[3], z, shade = R2X_SV_AMBIENT;
            pixel_ray(q, k, x, y, O, D);
            if (ell_hit(q, E, O, D, z)) {   // always, for the id that won the pixel
                double v[3], m[3], n[3];
                for (int i = 0; i < 3; ++i) v[i] = dsub(dadd(O[i], dmul(z, D[i])), E.c[i]);
                ell_local(E, v, m);
                for (int j = 0; j < 3; ++j) m[j] = dmul(m[j], E.k[j]);
                for (int i = 0; i < 3; ++i)
                    n[i] = dadd(dadd(dmul(E.R[i][0], m[0]), dmul(E.R[i][1], m[1])), dmul(E.R[i][2], m[2]));
                shade = headlight(n, D);
            }
            for (int i = 0; i < 3; ++i) out[i] = __double2float_rn(dmul((double)__ldg(at + i), shade));
        } else {
            const Cam k = load_cam(cameras, frame);
            const double* X = pos + (size_t)id * 9;
            double V[3][3];
            for (int v = 0; v < 3; ++v) to_cam(k, X + 3 * v, V[v]);
            double e1[3], e2[3], n[3];
            for (int i = 0; i < 3; ++i) {
                e1[i] = dsub(V[1][i], V[0][i]);
                e2[i] = dsub(V[2][i], V[0][i]);
            }
            n[0] = dsub(dmul(e1[1], e2[2]), dmul(e1[2], e2[1]));
            n[1] = dsub(dmul(e1[2], e2[0]), dmul(e1[0], e2[2]));
            n[2] = dsub(dmul(e1[0], e2[1]), dmul(e1[1], e2[0]));
            const double c = dot3(n, V[0]);
            double a, b;
            pixel_ab(q, k, x, y, a, b);
            double z = q.parallel ? ddiv(dsub(dsub(c, dmul(n[0], a)), dmul(n[1], b)), n[2])
                                  : ddiv(c, dadd(dadd(dmul(n[0], a), dmul(n[1], b)), n[2]));
            z = z >= q.near ? z : q.near;
            const double P[3] = {q.parallel ? a : dmul(a, z), q.parallel ? b : dmul(b, z), z};
            const double n2 = dot3(n, n);
            double w[3] = {1.0 / 3.0, 1.0 / 3.0, 1.0 / 3.0};
            if (n2 > 0.0) {
                for (int v = 0; v < 3; ++v) {   // w_v = n . ((V_{v+1} - P) x (V_{v+2} - P)) / |n|^2
                    const double* A = V[(v + 1) % 3];
                    const double* B = V[(v + 2) % 3];
                    const double s[3] = {dsub(A[0], P[0]), dsub(A[1], P[1]), dsub(A[2], P[2])};
                    const double t[3] = {dsub(B[0], P[0]), dsub(B[1], P[1]), dsub(B[2], P[2])};
                    const double cr[3] = {dsub(dmul(s[1], t[2]), dmul(s[2], t[1])),
                                          dsub(dmul(s[2], t[0]), dmul(s[0], t[2])),
                                          dsub(dmul(s[0], t[1]), dmul(s[1], t[0]))};
                    w[v] = ddiv(dot3(n, cr), n2);
                }
            }
            if (kind == R2X_SV_MESH) {
                double N[3];
                for (int i = 0; i < 3; ++i)
                    N[i] = dadd(dadd(dmul(w[0], (double)__ldg(at + 3 + i)), dmul(w[1], (double)__ldg(at + 6 + i))),
                                dmul(w[2], (double)__ldg(at + 9 + i)));
                double D[3];   // the headlight: along the pixel's ray, in world coordinates
                for (int i = 0; i < 3; ++i)
                    D[i] = q.parallel ? k.f[i] : dadd(dadd(k.f[i], dmul(a, k.r[i])), dmul(b, k.u[i]));
                const double shade = headlight(N, D);
                for (int i = 0; i < 3; ++i) out[i] = __double2float_rn(dmul((double)__ldg(at + i), shade));
            } else {   // textured
                const double tu = dadd(dadd(dmul(w[0], (double)__ldg(at + 3)), dmul(w[1], (double)__ldg(at + 5))),
                                       dmul(w[2], (double)__ldg(at + 7)));
                const double tv = dadd(dadd(dmul(w[0], (double)__ldg(at + 4)), dmul(w[1], (double)__ldg(at + 6))),
                                       dmul(w[2], (double)__ldg(at + 8)));
                const int j = (int)fmin(fmax(floor(dmul(tu, (double)q.tw)), 0.0), (double)(q.tw - 1));
                const int i = (int)fmin(fmax(floor(dmul(tv, (double)q.th)), 0.0), (double)(q.th - 1));
                const int ti = __ldg(meta + 2 * (size_t)id + 1);
                const float val = __ldg(tex + ((long long)ti * q.th + i) * q.tw + j);
                const float t = fminf(fmaxf(val, 0.0f), 1.0f);   // NaN -> 0
                if (q.K == 1) {
                    for (int c2 = 0; c2 < 3; ++c2) out[c2] = __ldg(lut + c2);
                } else {
                    const float ps = __fmul_rn(t, (float)(q.K - 1));
                    const int jj = min((int)floorf(ps), q.K - 2);
                    const float ww = __fsub_rn(ps, (float)jj);
                    for (int c2 = 0; c2 < 3; ++c2)
                        out[c2] = fblend(__ldg(lut + 3 * jj + c2), __ldg(lut + 3 * jj + 3 + c2), ww);
                }
            }
        }
    }
    float* o = rgb + px * 3;
    o[0] = out[0]; o[1] = out[1]; o[2] = out[2];
}

int bad(const char* what) {
    char msg[200];
    snprintf(msg, sizeof msg, "r2x_scene_raster: bad %s", what);
    return fail_msg(R2X_ERR_INVALID, msg);
}

size_t records_offset() { return 64; }

}  // namespace
}  // namespace r2x

extern "C" {

size_t r2x_scene_raster_scratch_bytes(int n_prims, int n_frames) {
    if (n_prims < 1 || n_frames < 1 || (long long)n_prims * n_frames > 2147483647ll) return 0;
    return r2x::records_offset() + (size_t)n_prims * n_frames * sizeof(r2x::SvRecord);
}

int r2x_scene_raster(void* stream, int n_prims, const double* pos, const int* meta, const float* attr, int n_tex,
                     int tex_h, int tex_w, const float* tex, const float* lut, int K, int n_frames, int H, int W,
                     const float* cameras, int parallel, double near, const float* background,
                     unsigned long long* keys, float* rgb, void* scratch, size_t scratch_bytes) {
    using namespace r2x;
    if (!pos || !meta || !attr || !lut || !cameras || !background || !keys || !rgb || !scratch)
        return bad("pointer (NULL)");
    if (n_prims < 1) return bad("n_prims (>= 1)");
    if (n_frames < 1 || n_frames > SV_MAX_GRID) return bad("n_frames (1 to 65535)");
    if ((long long)n_prims * n_frames > 2147483647ll)
        return bad("n_prims (n_prims * n_frames must be <= 2^31 - 1)");
    if (H < 1 || W < 1 || H > R2X_SV_MAX_SIDE || W > R2X_SV_MAX_SIDE) return bad("image (H and W from 1 to 16384)");
    if (n_tex < 0) return bad("n_tex (>= 0)");
    if (n_tex > 0) {
        if (!tex) return bad("pointer (tex is NULL with n_tex > 0)");
        if (tex_h < 1 || tex_w < 1 || tex_h > R2X_SV_MAX_SIDE || tex_w > R2X_SV_MAX_SIDE)
            return bad("texture (tex_h and tex_w from 1 to 16384)");
        if ((long long)n_tex * tex_h * tex_w > 2147483647ll) return bad("texture (n_tex * tex_h * tex_w <= 2^31 - 1)");
    }
    if (K < 1 || K > 4096) return bad("K (1 to 4096 LUT entries)");
    if (parallel != 0 && parallel != 1) return bad("parallel (0 or 1)");
    if (!std::isfinite(near) || !(near > 0.0)) return bad("near (finite, > 0)");
    for (int c = 0; c < 3; ++c)
        if (!std::isfinite(background[c])) return bad("background (finite)");
    if (scratch_bytes < r2x_scene_raster_scratch_bytes(n_prims, n_frames)) return bad("scratch (too small)");

    SvParams q;
    q.n_prims = n_prims; q.n_frames = n_frames; q.H = H; q.W = W; q.parallel = parallel;
    q.n_tex = n_tex; q.th = n_tex ? tex_h : 1; q.tw = n_tex ? tex_w : 1; q.K = K; q.near = near;
    for (int c = 0; c < 3; ++c) q.bg[c] = background[c];
    cudaStream_t st = (cudaStream_t)stream;
    SvCounters* cnt = (SvCounters*)scratch;
    SvRecord* rec = (SvRecord*)((char*)scratch + records_offset());
    R2X_CUDA_OK(cudaMemsetAsync(cnt, 0, sizeof(SvCounters), st));
    R2X_CUDA_OK(cudaMemsetAsync(keys, 0xff, (size_t)n_frames * H * W * sizeof(unsigned long long), st));
    sv_setup_kernel<<<dim3((unsigned)((n_prims + 255) / 256), 1, (unsigned)n_frames), 256, 0, st>>>(
        q, pos, meta, attr, cameras, keys, cnt, rec);
    R2X_CUDA_OK(cudaGetLastError());
    sv_scan_kernel<<<1, SV_SCAN_THREADS, 0, st>>>(cnt, rec);
    R2X_CUDA_OK(cudaGetLastError());
    sv_tile_kernel<<<SV_TILE_CTAS, dim3(SV_TILE, SV_TILE), 0, st>>>(q, pos, meta, attr, cameras, keys, cnt, rec);
    R2X_CUDA_OK(cudaGetLastError());
    const dim3 grid((unsigned)((W + SV_TILE - 1) / SV_TILE), (unsigned)((H + SV_TILE - 1) / SV_TILE),
                    (unsigned)n_frames);
    sv_resolve_kernel<<<grid, dim3(SV_TILE, SV_TILE), 0, st>>>(q, pos, meta, attr, tex, lut, cameras, keys, rgb);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
