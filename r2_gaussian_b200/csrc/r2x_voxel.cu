// r2x_voxel.cu -- density-volume (3-D voxelizer) kernels for sm_90a.
//
// Replaces the reference's VOX/forward.cu (preprocessCUDA :58-178, renderCUDA :183-315) and
// VOX/backward.cu (renderCUDA :216-374, computeCov3DCUDA :86-177, preprocessCUDA :180-213).
//
// Same machinery as r2x_raster.cu with 8x8x8 tiles:
//   voxel_preprocess_kernel  per Gaussian, TMA-staged parameters, bit-exact radii / cube / tiles_touched.
//   voxel_render_kernel      persistent CTAs pull (tile, chunk of <= 256 instances) work items from the atomic
//                            queue of the work plan; 256 threads = 4 list slices x 64 (x,y) columns; each thread
//                            owns the 8 voxels of a z column (contiguous in memory): the x/y part of the
//                            quadratic form is computed once per Gaussian and column, the z part runs by
//                            forward differences (exact Horner path for flagged Gaussians).
//   voxel_render_bwd_kernel  one thread per (tile, Gaussian) instance, loops over the 512 voxels and keeps
//                            the ten weighted moments in registers; no atomics; emission-order slots.
//   voxel_gauss_bwd_kernel   per Gaussian: fixed-order sum of its (contiguous) instance moments + chain rule.
#include "r2x_voxel.cuh"

namespace r2x {

static constexpr float LOG2E = 1.4426950408889634f;

struct VoxCov {
    float a, b, c, d, e, f;  // covariance in voxel units
    float det;
};

// hat = D Sigma D with D = diag(1/dVoxel) and its determinant; bit-exact restatement of the dataflow
// nvcc produced for VOX/forward.cu:110-125.
__device__ __forceinline__ VoxCov voxel_cov(const float* c3, float ix, float iy, float iz) {
    VoxCov v;
    v.a = fmul(fmul(ix, c3[0]), ix);
    v.b = fmul(fmul(iy, c3[1]), ix);
    v.c = fmul(fmul(iz, c3[2]), ix);
    v.d = fmul(fmul(iy, c3[3]), iy);
    v.e = fmul(fmul(iz, c3[4]), iy);
    v.f = fmul(fmul(iz, c3[5]), iz);
    const float ad = fmul(v.a, v.d), ae = fmul(v.a, v.e), bf = fmul(v.b, v.f), cd = fmul(v.c, v.d);
    float det = fmul(ad, v.f);
    det = ffma(fmul(fadd(v.b, v.b), v.c), v.e, det);
    det = ffma(-v.e, ae, det);
    det = ffma(-v.b, bf, det);
    det = ffma(-v.c, cd, det);
    v.det = det;
    return v;
}

__device__ __forceinline__ void voxel_inverse(const VoxCov& v, float* inv) {
    const float di = frcp(v.det);
    const float ad = fmul(v.a, v.d), ae = fmul(v.a, v.e), bf = fmul(v.b, v.f), cd = fmul(v.c, v.d);
    inv[0] = fmul(ffma(v.d, v.f, -fmul(v.e, v.e)), di);
    inv[1] = fmul(ffma(v.c, v.e, -bf), di);
    inv[2] = fmul(ffma(v.b, v.e, -cd), di);
    inv[3] = fmul(ffma(v.a, v.f, -fmul(v.c, v.c)), di);
    inv[4] = fmul(ffma(v.b, v.c, -ae), di);
    inv[5] = fmul(ffma(-v.b, v.b, ad), di);
}

constexpr int VPRE_THREADS = 256;

__global__ void __launch_bounds__(VPRE_THREADS) voxel_preprocess_kernel(
    int P, const float* __restrict__ means, const float* __restrict__ scales, float scale_modifier,
    const float* __restrict__ rots, const float* __restrict__ opac, const float* __restrict__ cov3D_precomp,
    VoxelGrid vg, int use_tma, int* __restrict__ radii_x, int* __restrict__ radii_y, int* __restrict__ radii_z,
    VoxelGeom geom, DirectBin db, int direct, Activation act) {
    extern __shared__ __align__(16) uint32_t s_hist[];   // [T] when direct binning
    __shared__ __align__(16) float s_means[VPRE_THREADS * 3];
    __shared__ __align__(16) float s_scales[VPRE_THREADS * 3];
    __shared__ __align__(16) float4 s_rots[VPRE_THREADS];
    __shared__ __align__(16) float s_opac[VPRE_THREADS];
    __shared__ __align__(8) uint64_t s_bar;

    const int tid = threadIdx.x;
    const int base = blockIdx.x * VPRE_THREADS;
    const int g = base + tid;
    const bool full = (base + VPRE_THREADS <= P);
    const bool tma = use_tma && full;
    if (tma && tid == 0) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
        mbar_expect_tx(&s_bar, VPRE_THREADS * (12 + 4 + 12 + 16));
        tma_load_1d(s_means, means + (size_t)base * 3, VPRE_THREADS * 12, &s_bar);
        tma_load_1d(s_opac, opac + base, VPRE_THREADS * 4, &s_bar);
        tma_load_1d(s_scales, scales + (size_t)base * 3, VPRE_THREADS * 12, &s_bar);
        tma_load_1d(s_rots, rots + (size_t)base * 4, VPRE_THREADS * 16, &s_bar);
    }
    __syncthreads();
    if (tma) mbar_wait(&s_bar, 0);
    const bool live = g < P;

    float mx = 0.f, my = 0.f, mz = 0.f, s0 = 0.f, s1 = 0.f, s2 = 0.f, rho = 0.f;
    float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
    if (!live) {
    } else if (tma) {
        mx = s_means[3 * tid]; my = s_means[3 * tid + 1]; mz = s_means[3 * tid + 2];
        rho = s_opac[tid];
        s0 = s_scales[3 * tid]; s1 = s_scales[3 * tid + 1]; s2 = s_scales[3 * tid + 2];
        q = s_rots[tid];
    } else {
        mx = means[3 * (size_t)g]; my = means[3 * (size_t)g + 1]; mz = means[3 * (size_t)g + 2];
        rho = opac[g];
        // the reference reads scales unconditionally (VOX/forward.cu:137): the radius needs them even
        // when a precomputed covariance is supplied
        s0 = scales[3 * (size_t)g]; s1 = scales[3 * (size_t)g + 1]; s2 = scales[3 * (size_t)g + 2];
        q = rots ? make_float4(rots[4 * (size_t)g], rots[4 * (size_t)g + 1], rots[4 * (size_t)g + 2], rots[4 * (size_t)g + 3])
                 : make_float4(1.f, 0.f, 0.f, 0.f);
    }
    if (act.enabled && live) {      // raw parameters: apply the activations here
        rho = act_softplus(rho);
        s0 = act_scale(act, s0); s1 = act_scale(act, s1); s2 = act_scale(act, s2);
        float nrm;
        q = act_normalize(q, nrm);
    }
    int rxi = 0, ryi = 0, rzi = 0;
    uint32_t ntiles = 0, c01 = 0, c23 = 0, c45 = 0;
    float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0, r2 = r0;
    float depth_out = 0.f;

    float c3[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (!live) {
    } else if (cov3D_precomp) {
#pragma unroll
        for (int k = 0; k < 6; ++k) c3[k] = cov3D_precomp[6 * (size_t)g + k];
    } else {
        cov3d_from_scale_rot(s0, s1, s2, scale_modifier, q, c3);
    }
    const VoxCov vc = voxel_cov(c3, vg.ix, vg.iy, vg.iz);
    if (live && vc.det != 0.0f) {
        float inv[6];
        voxel_inverse(vc, inv);
        const float ms3 = fmul(fmaxf(fmaxf(s0, s1), s2), 3.0f);
        const float rx = ceilf(fdiv(ms3, vg.dvx)), ry = ceilf(fdiv(ms3, vg.dvy)), rz = ceilf(fdiv(ms3, vg.dvz));
        const float pvx = fdiv(ffma(vg.sx, 0.5f, fsub(mx, vg.cx)), vg.dvx);
        const float pvy = fdiv(ffma(vg.sy, 0.5f, fsub(my, vg.cy)), vg.dvy);
        const float pvz = fdiv(ffma(vg.sz, 0.5f, fsub(mz, vg.cz)), vg.dvz);
        const float hx = fadd(pvx, rx), hy = fadd(pvy, ry), hz = fadd(pvz, rz);
        const float lx = fsub(pvx, rx), ly = fsub(pvy, ry), lz = fsub(pvz, rz);
        const bool outside = (hx < 0.f) || (hy < 0.f) || (hz < 0.f) || (lx > (float)vg.nx) || (ly > (float)vg.ny) ||
                             (lz > (float)vg.nz);
        if (!outside) {
            const int x0 = min(vg.gx, max(0, (int)fmul(lx, 0.125f)));
            const int y0 = min(vg.gy, max(0, (int)fmul(ly, 0.125f)));
            const int z0 = min(vg.gz, max(0, (int)fmul(lz, 0.125f)));
            const int x1 = min(vg.gx, max(0, (int)fmul(fadd(fadd(hx, 8.0f), -1.0f), 0.125f)));
            const int y1 = min(vg.gy, max(0, (int)fmul(fadd(fadd(hy, 8.0f), -1.0f), 0.125f)));
            const int z1 = min(vg.gz, max(0, (int)fmul(fadd(fadd(hz, 8.0f), -1.0f), 0.125f)));
            const int nt = (x1 - x0) * (y1 - y0) * (z1 - z0);
            if (nt != 0) {
                rxi = (int)rx; ryi = (int)ry; rzi = (int)rz;
                ntiles = (uint32_t)nt;
                // exponent-2 domain (see r2x_raster.cu): q = -power*log2(e) - log2(rho), alpha = 2^-q,
                // alpha >= 1e-6 <=> q <= log2(1e6).  r2.w = 0: fast path (forward differences along z, no
                // power test -- valid for a positive-definite conic); r2.w = rho: exact path.
                const float lw = (rho > 0.0f) ? (float)log2((double)rho) : -__int_as_float(0x7f800000);
                const float F2 = inv[5] * (0.5f * LOG2E);
                const float m01 = inv[0] * inv[3] - inv[1] * inv[1];
                const float det3 = inv[0] * (inv[3] * inv[5] - inv[4] * inv[4]) - inv[1] * (inv[1] * inv[5] - inv[4] * inv[2]) +
                                   inv[2] * (inv[1] * inv[4] - inv[3] * inv[2]);
                const bool pd = (inv[0] > 0.0f) && (inv[3] > 0.0f) && (inv[5] > 0.0f) && (m01 > 1e-4f * inv[0] * inv[3]) &&
                                (det3 > 1e-4f * inv[0] * inv[3] * inv[5]);
                const bool fast = !(rho > 0.0f) || (pd && F2 <= 2.0f && lw <= 20.0f && lw >= -100.0f);
                r0 = make_float4(pvx, pvy, pvz, lw);
                r1 = make_float4(inv[0] * (0.5f * LOG2E), inv[1] * LOG2E, inv[2] * LOG2E, inv[3] * (0.5f * LOG2E));
                // r2.z = K = 2^(-2 F2): ratio of the multiplicative forward differences along z (voxel_fast_8)
                r2 = make_float4(inv[4] * LOG2E, F2, (float)exp2(-2.0 * (double)F2), fast ? 0.0f : rho);
                depth_out = mz;
                c01 = (uint32_t)x0 | ((uint32_t)y0 << 16);
                c23 = (uint32_t)z0 | ((uint32_t)x1 << 16);
                c45 = (uint32_t)y1 | ((uint32_t)z1 << 16);
            }
        }
    }
    if (live) {
        radii_x[g] = rxi; radii_y[g] = ryi; radii_z[g] = rzi;
        geom.tiles_touched[g] = ntiles;
        geom.rec[4 * (size_t)g + 0] = r0;
        geom.rec[4 * (size_t)g + 1] = r1;
        geom.rec[4 * (size_t)g + 2] = r2;
        geom.rec[4 * (size_t)g + 3] = make_float4(rho, depth_out, 0.f, 0.f);   // backward / export only (never gathered)
        uint32_t* cu = reinterpret_cast<uint32_t*>(geom.cube + 6 * (size_t)g);
        cu[0] = c01; cu[1] = c23; cu[2] = c45;
    }
    if (direct) block_tile_histogram(s_hist, db, c01, c23, c45, ntiles, vg.gx, vg.gy);
}

// ------------------------------------------------------------------------------------------------
// forward render: persistent CTAs pull (tile, chunk) work items from the atomic queue of r2x_binning.cuh
// ------------------------------------------------------------------------------------------------
constexpr int VR_THREADS = 256;
constexpr int VR_SLICES = 4;
static_assert(PLAN_CHUNK == VR_THREADS, "one staged record per thread");

struct VWorkItem {
    int tile, chunk, nch, n;
    uint32_t begin;
    bool valid;
};

__device__ __forceinline__ VWorkItem vfetch_item(const TilePlan& pl, const uint2* __restrict__ ranges, uint32_t item,
                                                 uint32_t total) {
    VWorkItem w;
    w.valid = item < total;
    w.tile = 0; w.chunk = 0; w.nch = 1; w.n = 0; w.begin = 0;
    if (w.valid) plan_decode(pl, ranges, item, w.tile, w.chunk, w.nch, w.begin, w.n);
    return w;
}

constexpr float VQ_CUT = 19.931568569324174f;   // log2(1e6): alpha = 2^-q >= 1e-6  <=>  q <= VQ_CUT

// acc += e  iff  e >= 1e-6   (FSETP + predicated FADD; a NaN never passes)
__device__ __forceinline__ void vadd_if_alpha(float& acc, float e) {
    asm("{\n"
        ".reg .pred p;\n"
        "setp.ge.f32 p, %1, 0f358637BD;\n"
        "@p add.f32 %0, %0, %1;\n"
        "}\n"
        : "+f"(acc)
        : "f"(e));
}

// 8 voxels of one z column.  q(k) = q0 + lin*dz + F2*dz^2 - log2 rho with dz = dz0 - k has constant second
// differences along z, so alpha(k) = 2^-q(k) advances by multiplicative forward differences exactly as in
// r2x_raster.cu::render_fast_8: alpha(k+1) = alpha(k) D(k), D(k+1) = D(k) K, K = 2^(-2 F2) = r2.z; runs of 4 voxels,
// the column's two runs packed in register pairs (pack2 / mul2); the reference's alpha < 1e-6 skip is tested on alpha itself.
__device__ __forceinline__ void voxel_fast_8(float (&acc)[8], const float4 r0, const float4 r1, const float4 r2,
                                             float fx, float fy, float fz0) {
    const float dx = r0.x - fx, dy = r0.y - fy, dz0 = r0.z - fz0;
    const float q0 = fmaf(dx, fmaf(r1.x, dx, r1.y * dy), fmaf(r1.w * dy, dy, -r0.w));
    const float lin = fmaf(r1.z, dx, r2.x * dy);
    const float a2 = r2.y + r2.y;
    const float e0 = r2.y - lin;                      // d(k) = e0 - a2 (dz0 - k)
    const uint64_t DZ = pack2(dz0, dz0 - 4.0f);
    const uint64_t Q = fma2(DZ, fma2(pack2(r2.y, r2.y), DZ, pack2(lin, lin)), pack2(q0, q0));
    const uint64_t Dd = fma2(pack2(-a2, -a2), DZ, pack2(e0, e0));
    float qa, qb, da, db, ea, eb;
    unpack2(Q, qa, qb);
    unpack2(Dd, da, db);
    uint64_t E = pack2(ex2_approx(-qa), ex2_approx(-qb)), D = pack2(ex2_approx(-da), ex2_approx(-db));
    const uint64_t K = pack2(r2.z, r2.z);
    unpack2(E, ea, eb);
    vadd_if_alpha(acc[0], ea);
    vadd_if_alpha(acc[4], eb);
#pragma unroll
    for (int k = 1; k < 4; ++k) {
        E = mul2(E, D);
        if (k < 3) D = mul2(D, K);
        unpack2(E, ea, eb);
        vadd_if_alpha(acc[k], ea);
        vadd_if_alpha(acc[4 + k], eb);
    }
}

__device__ __forceinline__ void voxel_exact_8(float (&acc)[8], const float4 r0, const float4 r1, const float4 r2,
                                              float fx, float fy, float fz0) {
    const float dx = r0.x - fx, dy = r0.y - fy, dz0 = r0.z - fz0;
    const float q0 = fmaf(dx, fmaf(r1.x, dx, r1.y * dy), (r1.w * dy) * dy);
    const float lin = fmaf(r1.z, dx, r2.x * dy);
    const float qmax = VQ_CUT + r0.w;
    const uint32_t lim = (qmax >= 0.0f) ? (__float_as_uint(qmax) + 1u) : 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float dz = dz0 - (float)k;
        const float q = fmaf(dz, fmaf(r2.y, dz, lin), q0);   // = -power * log2(e)
        if (__float_as_uint(q) < lim) acc[k] = fmaf(r2.w, ex2_approx(-q), acc[k]);
    }
}

// A work item (tile, chunk) holds up to VOX_CHUNK_CAP instances; the CTA walks it in SEGMENTS of <= VR_THREADS records
// (what one staging buffer holds), keeps the 8 voxel sums of every thread in registers across the segments, and runs
// the epilogue (cross-slice reduction, store, multi-chunk arrival) once per item.  The stream of segments is
// double-buffered exactly like the items used to be: segment A computes while B's records land and C's ids are read.
struct VSeg {
    int tile, chunk, nch, n;
    uint32_t begin;
    bool valid, first, last;
};

__global__ void __launch_bounds__(VR_THREADS) voxel_render_kernel(VoxelGrid vg, const uint2* __restrict__ ranges,
                                                                  const uint32_t* __restrict__ point_list,
                                                                  const float4* __restrict__ rec, TilePlan pl,
                                                                  float* __restrict__ out_volume) {
    __shared__ __align__(16) float4 s_rec[2][VR_THREADS][3];      // 24 KB
    __shared__ __align__(16) float s_red[VR_SLICES - 1][64][8];   // 6 KB
    __shared__ uint32_t s_next;
    __shared__ uint32_t s_last;

    const int tid = threadIdx.x;
    const int slice = tid >> 6, q = tid & 63;
    const int lx = q >> 3, ly = q & 7;
    const uint32_t total = (uint32_t)pl.num_tiles + pl.extra_off[pl.num_tiles];

    // segment stream (all of it uniform across the CTA)
    VWorkItem it;
    it.valid = false; it.tile = 0; it.chunk = 0; it.nch = 1; it.n = 0; it.begin = 0;
    int handed = 0;          // instances of `it` already handed out
    bool has = false;        // `it` still has a segment to hand out
    uint32_t resv = 0, resv_end = 0;   // item indices reserved from the queue, not yet decoded
    auto refill = [&](uint32_t idx) {
        it = vfetch_item(pl, ranges, idx, total);
        handed = 0;
        has = it.valid;
    };
    auto take = [&]() {
        VSeg sg;
        sg.valid = has;
        sg.tile = it.tile; sg.chunk = it.chunk; sg.nch = it.nch;
        sg.begin = it.begin + (uint32_t)handed;
        const int rem = it.n - handed;
        sg.n = has ? (rem < VR_THREADS ? rem : VR_THREADS) : 0;
        sg.first = has && handed == 0;
        handed += sg.n;
        sg.last = has && handed >= it.n;
        if (sg.last) has = false;
        return sg;
    };

    if (tid == 0) s_next = atomicAdd(&pl.counter[0], 2u);
    __syncthreads();
    resv = s_next; resv_end = resv + 2;
    __syncthreads();
    refill(resv++);
    VSeg A = take();
    if (!has) refill(resv++);
    VSeg B = take();
    uint32_t idB = 0;
    if (A.valid && tid < A.n) {
        const uint32_t id = point_list[A.begin + tid];
        cp_async16(&s_rec[0][tid][0], &rec[4 * (size_t)id]);
        cp_async16(&s_rec[0][tid][1], &rec[4 * (size_t)id + 1]);
        cp_async16(&s_rec[0][tid][2], &rec[4 * (size_t)id + 2]);
    }
    cp_async_commit();
    if (B.valid && tid < B.n) idB = point_list[B.begin + tid];
    int stage = 0;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;

    while (A.valid) {
        const bool need_atomic = !has && resv >= resv_end;
        if (need_atomic && tid == 0) s_next = atomicAdd(&pl.counter[0], 1u);
        if (B.valid && tid < B.n) {
            cp_async16(&s_rec[stage ^ 1][tid][0], &rec[4 * (size_t)idB]);
            cp_async16(&s_rec[stage ^ 1][tid][1], &rec[4 * (size_t)idB + 1]);
            cp_async16(&s_rec[stage ^ 1][tid][2], &rec[4 * (size_t)idB + 2]);
        }
        cp_async_commit();
        cp_async_wait<1>();
        const int any_exact = __syncthreads_or((tid < A.n) && (s_rec[stage][tid][2].w != 0.0f));
        if (!has) refill(resv < resv_end ? resv++ : s_next);
        VSeg Cw = take();
        uint32_t idC = 0;
        if (Cw.valid && tid < Cw.n) idC = point_list[Cw.begin + tid];

        const int tx = A.tile % vg.gx, ty = (A.tile / vg.gx) % vg.gy, tz = A.tile / (vg.gx * vg.gy);
        const float fx = (float)(tx * R2X_VTILE + lx) + 0.5f;
        const float fy = (float)(ty * R2X_VTILE + ly) + 0.5f;
        const float fz0 = (float)(tz * R2X_VTILE) + 0.5f;
        if (A.first) {
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        }
        if (!any_exact) {
#pragma unroll 2
            for (int j = slice; j < A.n; j += VR_SLICES)
                voxel_fast_8(acc, s_rec[stage][j][0], s_rec[stage][j][1], s_rec[stage][j][2], fx, fy, fz0);
        } else {
            for (int j = slice; j < A.n; j += VR_SLICES) {
                const float4 r0 = s_rec[stage][j][0], r1 = s_rec[stage][j][1], r2 = s_rec[stage][j][2];
                if (r2.w == 0.0f) voxel_fast_8(acc, r0, r1, r2, fx, fy, fz0);
                else voxel_exact_8(acc, r0, r1, r2, fx, fy, fz0);
            }
        }
        if (A.last) {
            if (slice > 0) {
#pragma unroll
                for (int k = 0; k < 8; ++k) s_red[slice - 1][q][k] = acc[k];
            }
            __syncthreads();
            const int x = tx * R2X_VTILE + lx, y = ty * R2X_VTILE + ly, z0 = tz * R2X_VTILE;
            const bool col_in = (x < vg.nx && y < vg.ny);
            float* dst = out_volume + ((size_t)x * vg.ny + y) * vg.nz + z0;
            if (slice == 0) {
                float v[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    v[k] = acc[k];
                    v[k] += s_red[0][q][k];
                    v[k] += s_red[1][q][k];
                    v[k] += s_red[2][q][k];
                }
                if (A.chunk == 0) {
                    if (col_in) {
#pragma unroll
                        for (int k = 0; k < 8; ++k)
                            if (z0 + k < vg.nz) dst[k] = v[k];
                    }
                } else {
                    const size_t slot = (size_t)(pl.extra_off[A.tile] + A.chunk - 1);
                    float4* ps = reinterpret_cast<float4*>(&pl.partial[slot * 512 + q * 8]);
                    ps[0] = make_float4(v[0], v[1], v[2], v[3]);
                    ps[1] = make_float4(v[4], v[5], v[6], v[7]);
                }
            }
            if (A.nch > 1) {
                __threadfence();
                __syncthreads();
                if (tid == 0) s_last = (atomicAdd(&pl.tile_done[A.tile], 1u) == (uint32_t)(A.nch - 1)) ? 1u : 0u;
                __syncthreads();
                if (s_last) {
                    __threadfence();
                    if (slice == 0 && col_in) {
                        const size_t base = (size_t)pl.extra_off[A.tile];
                        float v[8];
#pragma unroll
                        for (int k = 0; k < 8; ++k) v[k] = (z0 + k < vg.nz) ? __ldcg(&dst[k]) : 0.f;
                        for (int c = 1; c < A.nch; ++c) {
                            const float4* ps = reinterpret_cast<const float4*>(&pl.partial[(base + c - 1) * 512 + q * 8]);
                            const float4 p0 = __ldcg(ps), p1 = __ldcg(ps + 1);
                            v[0] += p0.x; v[1] += p0.y; v[2] += p0.z; v[3] += p0.w;
                            v[4] += p1.x; v[5] += p1.y; v[6] += p1.z; v[7] += p1.w;
                        }
#pragma unroll
                        for (int k = 0; k < 8; ++k)
                            if (z0 + k < vg.nz) dst[k] = v[k];
                    }
                }
            }
        } else {
            __syncthreads();   // every thread is done with s_rec[stage] before the next segment's records land in it
        }
        A = B; B = Cw; idB = idC; stage ^= 1;
    }
}

// ------------------------------------------------------------------------------------------------
// backward render: thread = instance; moments S0, Sx,Sy,Sz, Sxx,Sxy,Sxz,Syy,Syz,Szz of t = dL*G
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) voxel_render_bwd_kernel(VoxelGrid vg, const uint2* __restrict__ ranges,
                                                               const uint32_t* __restrict__ point_list,
                                                               const uint32_t* __restrict__ inst_pos, VoxelGeom geom,
                                                               const float4* __restrict__ rec, TilePlan pl,
                                                               const float* __restrict__ dL_dvol,
                                                               float4* __restrict__ inst_grad) {
    __shared__ __align__(16) float s_dl[R2X_VTILE][R2X_VTILE][R2X_VTILE];
    __shared__ uint32_t s_next;
    const int tid = threadIdx.x;
    const uint32_t total = (uint32_t)pl.num_tiles + pl.extra_off[pl.num_tiles];
    int cur_tile = -1;
    while (true) {
        __syncthreads();
        if (tid == 0) s_next = atomicAdd(&pl.counter[1], 1u);
        __syncthreads();
        const uint32_t item = s_next;
        if (item >= total) break;
        int tile, chunk, nch, n;
        uint32_t begin;
        plan_decode(pl, ranges, item, tile, chunk, nch, begin, n);
        if (n == 0) continue;
        const int tx = tile % vg.gx, ty = (tile / vg.gx) % vg.gy, tz = tile / (vg.gx * vg.gy);
        if (tile != cur_tile) {
            for (int v = tid; v < 512; v += 256) {
                const int lz = v & 7, ly = (v >> 3) & 7, lx = v >> 6;
                const int x = tx * R2X_VTILE + lx, y = ty * R2X_VTILE + ly, z = tz * R2X_VTILE + lz;
                s_dl[lx][ly][lz] = (x < vg.nx && y < vg.ny && z < vg.nz) ? dL_dvol[((size_t)x * vg.ny + y) * vg.nz + z] : 0.f;
            }
            cur_tile = tile;
        }
        __syncthreads();
        for (int ii = tid; ii < n; ii += 256) {   // an item holds up to VOX_CHUNK_CAP instances: 256 per sweep
        const float fx0 = (float)(tx * R2X_VTILE) + 0.5f, fy0 = (float)(ty * R2X_VTILE) + 0.5f,
                    fz0 = (float)(tz * R2X_VTILE) + 0.5f;
        const uint32_t s = begin + (uint32_t)ii;
        const uint32_t g = point_list[s];
        const float4 r0 = rec[4 * (size_t)g];
        const float4 r1 = rec[4 * (size_t)g + 1];
        const float4 r2 = rec[4 * (size_t)g + 2];
        float S0 = 0.f, Sx = 0.f, Sy = 0.f, Sz = 0.f, Sxx = 0.f, Sxy = 0.f, Sxz = 0.f, Syy = 0.f, Syz = 0.f, Szz = 0.f;
        const float qmax = VQ_CUT + r0.w;   // contributes iff 0 <= q <= log2(rho / 1e-6)
        const uint32_t lim = (qmax >= 0.0f) ? (__float_as_uint(qmax) + 1u) : 0u;
        const float dz0 = r0.z - fz0;
        const bool fast = (r2.w == 0.0f);
        const float a2 = r2.y + r2.y;
        const float gcut = ex2_approx(-qmax);     // alpha = rho G >= 1e-6  <=>  G >= 2^-(VQ_CUT + log2 rho)
#pragma unroll 1
        for (int ix = 0; ix < R2X_VTILE; ++ix) {
            const float dx = r0.x - (fx0 + (float)ix);
            float X0 = 0.f, Xy = 0.f, Xyy = 0.f, Xz = 0.f, Xyz = 0.f, Xzz = 0.f;
#pragma unroll 1
            for (int iy = 0; iy < R2X_VTILE; ++iy) {
                const float dy = r0.y - (fy0 + (float)iy);
                const float q0 = fmaf(dx, fmaf(r1.x, dx, r1.y * dy), (r1.w * dy) * dy);
                const float lin = fmaf(r1.z, dx, r2.x * dy);
                const float4 da = *reinterpret_cast<const float4*>(&s_dl[ix][iy][0]);
                const float4 db = *reinterpret_cast<const float4*>(&s_dl[ix][iy][4]);
                const float dlv[8] = {da.x, da.y, da.z, da.w, db.x, db.y, db.z, db.w};
                float R0 = 0.f, Rz = 0.f, Rzz = 0.f;
                if (fast) {
                    // G(k) = 2^-quad(k) by multiplicative forward differences along z (voxel_fast_8); moments are taken
                    // about the voxel index k (immediates) and shifted to dz = dz0 - k afterwards
                    float N0 = 0.f, N1 = 0.f, N2 = 0.f;
#pragma unroll
                    for (int h4 = 0; h4 < 2; ++h4) {
                        const float dza = dz0 - (float)(4 * h4);
                        float G = ex2_approx(-fmaf(dza, fmaf(r2.y, dza, lin), q0));
                        float D = ex2_approx(-fmaf(-a2, dza, r2.y - lin));
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            if (k > 0) { G *= D; if (k < 3) D *= r2.z; }
                            const float t = (G >= gcut) ? dlv[4 * h4 + k] * G : 0.f;
                            N0 += t;
                            N1 = fmaf(t, (float)(4 * h4 + k), N1);
                            N2 = fmaf(t, (float)((4 * h4 + k) * (4 * h4 + k)), N2);
                        }
                    }
                    R0 = N0;
                    Rz = fmaf(dz0, N0, -N1);
                    Rzz = fmaf(dz0, fmaf(dz0, N0, -2.0f * N1), N2);
                } else {
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const float dz = dz0 - (float)k;
                        const float u = fmaf(r2.y, dz, lin);
                        const float qq = fmaf(dz, u, q0);
                        const float G = ex2_approx(-qq);
                        const float t = (__float_as_uint(qq) < lim) ? dlv[k] * G : 0.f;
                        R0 += t;
                        const float tdz = t * dz;
                        Rz += tdz;
                        Rzz = fmaf(tdz, dz, Rzz);
                    }
                }
                X0 += R0; Xz += Rz; Xzz += Rzz;
                Xy = fmaf(dy, R0, Xy);
                Xyy = fmaf(dy * dy, R0, Xyy);
                Xyz = fmaf(dy, Rz, Xyz);
            }
            S0 += X0; Sy += Xy; Sz += Xz; Syy += Xyy; Syz += Xyz; Szz += Xzz;
            Sx = fmaf(dx, X0, Sx);
            Sxx = fmaf(dx * dx, X0, Sxx);
            Sxy = fmaf(dx, Xy, Sxy);
            Sxz = fmaf(dx, Xz, Sxz);
        }
        // emission-order index: a Gaussian's instances are contiguous there
        const uint32_t slot = inst_pos ? inst_pos[s]
                                       : emission_slot(geom.cube, geom.offsets, geom.tiles_touched, g, (uint32_t)tx, (uint32_t)ty, (uint32_t)tz);
        inst_grad[3 * (size_t)slot] = make_float4(S0, Sx, Sy, Sz);
        inst_grad[3 * (size_t)slot + 1] = make_float4(Sxx, Sxy, Sxz, Syy);
        inst_grad[3 * (size_t)slot + 2] = make_float4(Syz, Szz, 0.f, 0.f);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// backward, per Gaussian
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) voxel_gauss_bwd_kernel(
    int P, const int* __restrict__ radii_x, const int* __restrict__ radii_y, const int* __restrict__ radii_z,
    const float* __restrict__ scales, float scale_modifier, const float* __restrict__ rots,
    const float* __restrict__ cov3D_precomp, VoxelGrid vg, VoxelGeom geom, long long capacity,
    const uint32_t* __restrict__ inst_pos,
    const float4* __restrict__ inst_grad, float* __restrict__ dL_dopacity, float* __restrict__ dL_dmean3D,
    float* __restrict__ dL_dcov3D, float* __restrict__ dL_dscale, float* __restrict__ dL_drot, Activation act) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P) return;
    const bool live = (radii_x[g] > 0) && (radii_y[g] > 0) && (radii_z[g] > 0);
    float dop = 0.f, dmean[3] = {0.f, 0.f, 0.f}, dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float ds[3] = {0.f, 0.f, 0.f}, dr[4] = {0.f, 0.f, 0.f, 0.f};
    if (live) {
        const uint32_t n = geom.tiles_touched[g];
        const uint32_t start = geom.offsets[g] - n;
        float S0 = 0.f, Sx = 0.f, Sy = 0.f, Sz = 0.f, Sxx = 0.f, Sxy = 0.f, Sxz = 0.f, Syy = 0.f, Syz = 0.f, Szz = 0.f;
        const uint32_t nlive = ((long long)start + n <= capacity) ? n : 0u;
#pragma unroll 4
        for (uint32_t k = 0; k < nlive; ++k) {
            const float4 a = inst_grad[3 * (size_t)(start + k)];
            const float4 b = inst_grad[3 * (size_t)(start + k) + 1];
            const float4 c = inst_grad[3 * (size_t)(start + k) + 2];
            S0 += a.x; Sx += a.y; Sy += a.z; Sz += a.w;
            Sxx += b.x; Sxy += b.y; Sxz += b.z; Syy += b.w;
            Syz += c.x; Szz += c.y;
        }
        const float rho = geom.rec[4 * (size_t)g + 3].x;
        const bool have_sr = (cov3D_precomp == nullptr);
        float s0 = 0.f, s1 = 0.f, s2 = 0.f;
        float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
        float c3[6];
        float raw_s[3] = {0.f, 0.f, 0.f}, qnorm = 1.f;
        if (have_sr) {
            s0 = scales[3 * (size_t)g]; s1 = scales[3 * (size_t)g + 1]; s2 = scales[3 * (size_t)g + 2];
            q = make_float4(rots[4 * (size_t)g], rots[4 * (size_t)g + 1], rots[4 * (size_t)g + 2], rots[4 * (size_t)g + 3]);
            if (act.enabled) {
                raw_s[0] = s0; raw_s[1] = s1; raw_s[2] = s2;
                s0 = act_scale(act, s0); s1 = act_scale(act, s1); s2 = act_scale(act, s2);
                q = act_normalize(q, qnorm);
            }
            cov3d_from_scale_rot(s0, s1, s2, scale_modifier, q, c3);
        } else {
#pragma unroll
            for (int k = 0; k < 6; ++k) c3[k] = cov3D_precomp[6 * (size_t)g + k];
        }
        const VoxCov vc = voxel_cov(c3, vg.ix, vg.iy, vg.iz);
        float inv[6];
        voxel_inverse(vc, inv);
        // VOX/backward.cu:348-370 with the per-pair sums factored into moments
        dop = act.enabled ? S0 * (1.0f - expf(-rho)) : S0;     // raw density: softplus' = 1 - exp(-rho)
        dmean[0] = rho * (-inv[0] * Sx - inv[1] * Sy - inv[2] * Sz) * vg.dvx;   // note: x dVoxel, as the reference
        dmean[1] = rho * (-inv[3] * Sy - inv[1] * Sx - inv[4] * Sz) * vg.dvy;
        dmean[2] = rho * (-inv[5] * Sz - inv[2] * Sx - inv[4] * Sy) * vg.dvz;
        const float ga = -0.5f * rho * Sxx, gb = -rho * Sxy, gc = -rho * Sxz, gd = -0.5f * rho * Syy, ge = -rho * Syz,
                    gf = -0.5f * rho * Szz;
        // conic3D = Sv^-1 (Sv = voxel-space covariance):  dL/dSv = -adj(Sv) G adj(Sv) / det^2, with the reference's
        // regularised 1 / (det^2 + 1e-7) (VOX/backward.cu:132-168); then Sv = D Sigma D, D = diag(1/dVoxel).
        const float sv[6] = {vc.a, vc.b, vc.c, vc.d, vc.e, vc.f};
        Mat3 K;
        const float det = sym_cofactors(sv, K);
        const float inv_det_sq = 1.0f / (det * det + 0.0000001f);
        if (inv_det_sq != 0.f) {
            const float g6[6] = {ga, gb, gc, gd, ge, gf};
            const Mat3 T = matmul<false, false>(K, matmul<false, false>(sym_grad_full(g6), K));
            float dh[6];
            sym_grad_pack(T, dh);
#pragma unroll
            for (int k = 0; k < 6; ++k) dh[k] *= -inv_det_sq;
            const float Mm[9] = {vg.ix, 0.f, 0.f, 0.f, vg.iy, 0.f, 0.f, 0.f, vg.iz};
            dcov3d_from_dhat(Mm, dh, dcov);
        }
        if (have_sr) {
            cov3d_backward(s0, s1, s2, scale_modifier, q, dcov, ds, dr);
            if (act.enabled) {
#pragma unroll
                for (int k = 0; k < 3; ++k) ds[k] *= act_scale_grad(act, raw_s[k]);
                act_normalize_grad(q, qnorm, dr);
            }
        }
    }
    dL_dopacity[g] = dop;
#pragma unroll
    for (int k = 0; k < 3; ++k) { dL_dmean3D[3 * (size_t)g + k] = dmean[k]; dL_dscale[3 * (size_t)g + k] = ds[k]; }
#pragma unroll
    for (int k = 0; k < 6; ++k) dL_dcov3D[6 * (size_t)g + k] = dcov[k];
#pragma unroll
    for (int k = 0; k < 4; ++k) dL_drot[4 * (size_t)g + k] = dr[k];
}

// ------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------
VoxelGrid make_voxel_grid(int nx, int ny, int nz, float sx, float sy, float sz, float cx, float cy, float cz) {
    VoxelGrid v;
    v.nx = nx; v.ny = ny; v.nz = nz;
    v.sx = sx; v.sy = sy; v.sz = sz;
    v.cx = cx; v.cy = cy; v.cz = cz;
    v.gx = (nx + R2X_VTILE - 1) / R2X_VTILE;
    v.gy = (ny + R2X_VTILE - 1) / R2X_VTILE;
    v.gz = (nz + R2X_VTILE - 1) / R2X_VTILE;
    // IEEE float32 divisions on the host == div.rn.f32 / rcp.rn.f32 on the device
    volatile float dvx = sx / (float)nx, dvy = sy / (float)ny, dvz = sz / (float)nz;
    v.dvx = dvx; v.dvy = dvy; v.dvz = dvz;
    volatile float ix = 1.0f / dvx, iy = 1.0f / dvy, iz = 1.0f / dvz;
    v.ix = ix; v.iy = iy; v.iz = iz;
    return v;
}

int launch_voxel_preprocess(cudaStream_t st, int P, const float* means, const float* scales, float scale_modifier,
                            const float* rots, const float* opac, const float* cov3D_precomp, const VoxelGrid& vg,
                            int* radii_x, int* radii_y, int* radii_z, const VoxelGeom& geom, const DirectBin* db) {
    if (P <= 0) return 0;
    auto al16 = [](const void* p) { return p && (((size_t)p) & 15) == 0; };
    const int use_tma = al16(means) && al16(opac) && al16(scales) && al16(rots);
    static_assert(VPRE_THREADS == DIRECT_BLOCK, "direct binning assumes one preprocess CTA per 256 Gaussians");
    const DirectBin dbv = db ? *db : DirectBin{};
    const size_t smem = db ? (size_t)db->num_tiles * sizeof(uint32_t) : 0;
    voxel_preprocess_kernel<<<(P + VPRE_THREADS - 1) / VPRE_THREADS, VPRE_THREADS, smem, st>>>(
        P, means, scales, scale_modifier, rots, opac, cov3D_precomp, vg, use_tma, radii_x, radii_y, radii_z, geom, dbv,
        db ? 1 : 0, current_activation());
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

static int vpersistent_grid(long long max_items, int sms) {
    const long long cap = sms * 4ll;   // 4 CTAs of 256 threads per SM (54 registers/thread)
    return (int)(max_items < cap ? (max_items > 0 ? max_items : 1) : cap);
}

int launch_voxel_render(cudaStream_t st, const VoxelGrid& vg, const VoxelGeom& geom, const uint2* ranges,
                        const uint32_t* point_list, const TilePlan& plan, long long R_launch, float* out_volume) {
    const long long items = (long long)plan.num_tiles + R_launch / PLAN_CHUNK + 1;
    int sms;
    R2X_CUDA_OK(sm_count(&sms));
    voxel_render_kernel<<<vpersistent_grid(items, sms), VR_THREADS, 0, st>>>(vg, ranges, point_list, geom.rec, plan,
                                                                        out_volume);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_voxel_render_bwd(cudaStream_t st, const VoxelGrid& vg, const VoxelGeom& geom, const uint2* ranges,
                            const uint32_t* point_list, const uint32_t* inst_pos, const TilePlan& plan,
                            long long R_launch, const float* dL_dvol, float4* inst_grad) {
    const long long items = (long long)plan.num_tiles + R_launch / PLAN_CHUNK + 1;
    int sms;
    R2X_CUDA_OK(sm_count(&sms));
    R2X_CUDA_OK(cudaMemsetAsync(plan.counter + 1, 0, sizeof(uint32_t), st));
    voxel_render_bwd_kernel<<<vpersistent_grid(items, sms), 256, 0, st>>>(vg, ranges, point_list, inst_pos, geom, geom.rec, plan,
                                                                     dL_dvol, inst_grad);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_voxel_gauss_bwd(cudaStream_t st, int P, const int* radii_x, const int* radii_y, const int* radii_z,
                           const float* scales, float scale_modifier, const float* rots, const float* cov3D_precomp,
                           const VoxelGrid& vg, const VoxelGeom& geom, long long capacity, const uint32_t* inst_pos,
                           const float4* inst_grad, float* dL_dopacity, float* dL_dmean3D, float* dL_dcov3D,
                           float* dL_dscale, float* dL_drot) {
    if (P <= 0) return 0;
    voxel_gauss_bwd_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, radii_x, radii_y, radii_z, scales, scale_modifier, rots,
                                                             cov3D_precomp, vg, geom, capacity, inst_pos, inst_grad, dL_dopacity,
                                                             dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot, current_activation());
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace r2x
