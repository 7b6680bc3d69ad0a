// Two-level direct binning for voxel grids with more tiles than the direct table can hold.
//
// The direct binning of r2x_binning.cu keeps a [Gaussian blocks][tiles] count table, which is what limits it to
// DIRECT_MAX_TILES tiles; a 256^3 query has 32768 tiles of 8^3 voxels and used to take the radix path (emit keys,
// two stable 8-bit passes, tile ranges: 0.64 of its 2.26 ms on 500k Gaussians).  Here the SAME direct machinery first
// bins the Gaussians into SUPERTILES of 4 x 4 x 4 tiles (level 1: at most DIRECT_MAX_TILES supertiles, i.e. grids up to
// 512^3), and a second level splits every supertile list -- cut into work items of at most L2_CHUNK entries by the
// level-1 work plan -- over the supertile's 64 tiles:
//
//   super_cube      per Gaussian: supertile cube + count, per-block supertile histogram row           (level 1)
//   direct_scan / direct_fill  (r2x_binning.cu)  -> ranges1[S], list1: Gaussian ids, ascending, per supertile
//   fine_count      per item: the 64 per-tile counts of its entries (one ballot per tile transposes the warp's
//                   32 x 64 membership matrix; a count is the population of a column)              -> table2[item][64]
//   fine_scan       per supertile: running prefix over its items, tile totals into tile_count[T]
//   scan            single-pass scan of tile_count in TILE-ID order (so the lists are tile-major like the reference's)
//   fine_ranges     ranges[t] = (start, end)
//   fine_fill       per item: rebuilds the same columns and writes every (entry, tile) id to
//                   start[t] + prefix[item][t] + rank of the entry among the item's entries on t
//
// Every list comes out ascending in Gaussian id -- the order the reference's stable sort produces -- so ranges and
// point_list are bit-identical to the radix path's (tests/test_voxel_gpu.py compares them).  No per-instance key,
// no sort, no inst_pos: the backward derives emission slots from offsets[] (emission_slot()).
// Scratch that would otherwise sit idle is reused: list1 = keys[0], extra rows of table2 = keys[1], the level-1
// extra-item list = vals[0] of the binning buffer.
#include <cstdlib>
#include <cstring>

#include "r2x_binning.cuh"

#define R2X_PASS(expr)               \
    do {                             \
        const int rc_ = (expr);      \
        if (rc_) return rc_;         \
    } while (0)

namespace r2x {

namespace {

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

constexpr int SUP = 4;               // tiles per supertile edge
constexpr int SUP_TILES = SUP * SUP * SUP;
constexpr int L2_CHUNK = PLAN_CHUNK; // level-1 entries per level-2 work item (== threads of the item's CTA)
static_assert(SUP_TILES == 64, "the membership of an entry is one 64-bit mask");
static_assert(L2_CHUNK == 256, "one thread per entry");

__device__ __forceinline__ void unpack_cube(const uint16_t* __restrict__ cube, uint32_t g, uint32_t& x0, uint32_t& y0,
                                            uint32_t& z0, uint32_t& x1, uint32_t& y1, uint32_t& z1) {
    const uint32_t* c = reinterpret_cast<const uint32_t*>(cube + 6 * (size_t)g);
    const uint32_t c01 = c[0], c23 = c[1], c45 = c[2];
    x0 = c01 & 0xffff; y0 = c01 >> 16; z0 = c23 & 0xffff; x1 = c23 >> 16; y1 = c45 & 0xffff; z1 = c45 >> 16;
}

// CTA b = Gaussians [256 b, 256 b + 256): supertile cube and count of every Gaussian, and row b of the level-1 table
__global__ void __launch_bounds__(DIRECT_BLOCK) super_cube_kernel(int P, const uint16_t* __restrict__ cube,
                                                                  const uint32_t* __restrict__ tiles_touched,
                                                                  uint16_t* __restrict__ cube1,
                                                                  uint32_t* __restrict__ tiles1, DirectBin db1, int gx1,
                                                                  int gy1) {
    extern __shared__ __align__(16) uint32_t s_hist[];
    const int g = blockIdx.x * DIRECT_BLOCK + threadIdx.x;
    uint32_t n1 = 0, p01 = 0, p23 = 0, p45 = 0;
    if (g < P) {
        if (tiles_touched[g]) {
            uint32_t x0, y0, z0, x1, y1, z1;
            unpack_cube(cube, (uint32_t)g, x0, y0, z0, x1, y1, z1);
            const uint32_t X0 = x0 / SUP, Y0 = y0 / SUP, Z0 = z0 / SUP;
            const uint32_t X1 = (x1 - 1) / SUP + 1, Y1 = (y1 - 1) / SUP + 1, Z1 = (z1 - 1) / SUP + 1;   // exclusive
            n1 = (X1 - X0) * (Y1 - Y0) * (Z1 - Z0);
            p01 = X0 | (Y0 << 16); p23 = Z0 | (X1 << 16); p45 = Y1 | (Z1 << 16);
        }
        uint32_t* c = reinterpret_cast<uint32_t*>(cube1 + 6 * (size_t)g);
        c[0] = p01; c[1] = p23; c[2] = p45;
        tiles1[g] = n1;
    }
    block_tile_histogram(s_hist, db1, p01, p23, p45, n1, gx1, gy1);
}

// which of supertile (sx, sy, sz)'s 64 tiles Gaussian g touches: bit (lz * 4 + ly) * 4 + lx
__device__ __forceinline__ unsigned long long local_mask(const uint16_t* __restrict__ cube, uint32_t g, uint32_t sx,
                                                         uint32_t sy, uint32_t sz) {
    uint32_t x0, y0, z0, x1, y1, z1;
    unpack_cube(cube, g, x0, y0, z0, x1, y1, z1);
    const uint32_t bx = sx * SUP, by = sy * SUP, bz = sz * SUP;
    const uint32_t lx0 = max(x0, bx) - bx, lx1 = min(x1, bx + SUP) - bx;
    const uint32_t ly0 = max(y0, by) - by, ly1 = min(y1, by + SUP) - by;
    const uint32_t lz0 = max(z0, bz) - bz, lz1 = min(z1, bz + SUP) - bz;
    const uint32_t xm = ((1u << lx1) - 1u) & ~((1u << lx0) - 1u);
    uint32_t plane = 0;
    for (uint32_t ly = ly0; ly < ly1; ++ly) plane |= xm << (SUP * ly);
    unsigned long long m = 0;
    for (uint32_t lz = lz0; lz < lz1; ++lz) m |= (unsigned long long)plane << (SUP * SUP * lz);
    return m;
}

// transposes the warp's 32 x 64 membership matrix: s_col[l] = ballot of "my entry touches local tile l"
__device__ __forceinline__ void warp_columns(unsigned long long mask, uint32_t* __restrict__ s_col_warp, int lane) {
    const uint32_t lo = (uint32_t)mask, hi = (uint32_t)(mask >> 32);
    uint32_t c_lo = 0, c_hi = 0;
#pragma unroll
    for (int l = 0; l < 32; ++l) {
        const uint32_t a = __ballot_sync(0xffffffffu, (lo >> l) & 1u);
        const uint32_t b = __ballot_sync(0xffffffffu, (hi >> l) & 1u);
        if (lane == l) { c_lo = a; c_hi = b; }
    }
    s_col_warp[lane] = c_lo;
    s_col_warp[lane + 32] = c_hi;
}

__device__ __forceinline__ uint32_t* table2_row(uint32_t* a, uint32_t* b, uint32_t item, int T1) {
    return item < (uint32_t)T1 ? a + (size_t)item * SUP_TILES : b + (size_t)(item - (uint32_t)T1) * SUP_TILES;
}

__global__ void __launch_bounds__(L2_CHUNK) fine_count_kernel(TilePlan pl1, const uint2* __restrict__ ranges1,
                                                              const uint32_t* __restrict__ list1,
                                                              const uint16_t* __restrict__ cube, int gx1, int gy1,
                                                              uint32_t* __restrict__ table2a,
                                                              uint32_t* __restrict__ table2b,
                                                              const uint32_t* __restrict__ status) {
    __shared__ uint32_t s_next;
    __shared__ uint32_t s_col[L2_CHUNK / 32][SUP_TILES];
    if (status[1]) return;     // the instance capacity is exceeded: nothing downstream is read
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t total = (uint32_t)pl1.num_tiles + pl1.extra_off[pl1.num_tiles];
    while (true) {
        __syncthreads();
        if (tid == 0) s_next = atomicAdd(&pl1.counter[0], 1u);
        __syncthreads();
        const uint32_t item = s_next;
        if (item >= total) break;
        int s, chunk, nch, n;
        uint32_t begin;
        plan_decode(pl1, ranges1, item, s, chunk, nch, begin, n);
        const uint32_t sx = (uint32_t)(s % gx1), sy = (uint32_t)((s / gx1) % gy1), sz = (uint32_t)(s / (gx1 * gy1));
        unsigned long long mask = 0;
        if (tid < n) mask = local_mask(cube, list1[begin + tid], sx, sy, sz);
        warp_columns(mask, s_col[warp], lane);
        __syncthreads();
        if (tid < SUP_TILES) {
            uint32_t c = 0;
#pragma unroll
            for (int w = 0; w < L2_CHUNK / 32; ++w) c += __popc(s_col[w][tid]);
            table2_row(table2a, table2b, item, pl1.num_tiles)[tid] = c;
        }
    }
}

// CTA = supertile, thread = local tile: counts of the supertile's items -> exclusive prefix over the items, total -> tile_count
__global__ void __launch_bounds__(SUP_TILES) fine_scan_kernel(TilePlan pl1, uint32_t* __restrict__ table2a,
                                                              uint32_t* __restrict__ table2b, int gx1, int gy1, int gx,
                                                              int gy, int gz, uint32_t* __restrict__ tile_count,
                                                              const uint32_t* __restrict__ status) {
    const int s = blockIdx.x, l = threadIdx.x;
    const uint32_t sx = (uint32_t)(s % gx1), sy = (uint32_t)((s / gx1) % gy1), sz = (uint32_t)(s / (gx1 * gy1));
    const uint32_t tx = sx * SUP + (l & 3), ty = sy * SUP + ((l >> 2) & 3), tz = sz * SUP + (l >> 4);
    const bool inside = tx < (uint32_t)gx && ty < (uint32_t)gy && tz < (uint32_t)gz;
    uint32_t run = 0;
    if (!status[1]) {
        const uint32_t e0 = pl1.extra_off[s], e1 = pl1.extra_off[s + 1];
        uint32_t* row = table2a + (size_t)s * SUP_TILES;
        uint32_t v = row[l];
        row[l] = 0;
        run = v;
        for (uint32_t e = e0; e < e1; ++e) {
            row = table2b + (size_t)e * SUP_TILES;
            v = row[l];
            row[l] = run;
            run += v;
        }
    }
    if (inside) tile_count[((size_t)tz * gy + ty) * gx + tx] = run;
}

__global__ void __launch_bounds__(256) fine_ranges_kernel(int T, const uint32_t* __restrict__ tile_count,
                                                          const uint32_t* __restrict__ tile_incl,
                                                          const uint32_t* __restrict__ status, uint2* __restrict__ ranges) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint32_t e = tile_incl[t], c = tile_count[t];
    ranges[t] = status[1] ? make_uint2(0u, 0u) : make_uint2(e - c, e);
}

__global__ void __launch_bounds__(L2_CHUNK) fine_fill_kernel(TilePlan pl1, const uint2* __restrict__ ranges1,
                                                             const uint32_t* __restrict__ list1,
                                                             const uint16_t* __restrict__ cube, int gx1, int gy1, int gx,
                                                             int gy, int gz, const uint32_t* __restrict__ table2a,
                                                             const uint32_t* __restrict__ table2b,
                                                             const uint32_t* __restrict__ tile_count,
                                                             const uint32_t* __restrict__ tile_incl,
                                                             const uint32_t* __restrict__ status,
                                                             uint32_t* __restrict__ point_list) {
    __shared__ uint32_t s_next;
    __shared__ uint32_t s_col[L2_CHUNK / 32][SUP_TILES];
    __shared__ uint32_t s_pre[L2_CHUNK / 32][SUP_TILES];
    if (status[1]) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t total = (uint32_t)pl1.num_tiles + pl1.extra_off[pl1.num_tiles];
    const uint32_t below = (1u << lane) - 1u;
    while (true) {
        __syncthreads();
        if (tid == 0) s_next = atomicAdd(&pl1.counter[1], 1u);
        __syncthreads();
        const uint32_t item = s_next;
        if (item >= total) break;
        int s, chunk, nch, n;
        uint32_t begin;
        plan_decode(pl1, ranges1, item, s, chunk, nch, begin, n);
        if (n == 0) continue;
        const uint32_t sx = (uint32_t)(s % gx1), sy = (uint32_t)((s / gx1) % gy1), sz = (uint32_t)(s / (gx1 * gy1));
        unsigned long long mask = 0;
        uint32_t g = 0;
        if (tid < n) {
            g = list1[begin + tid];
            mask = local_mask(cube, g, sx, sy, sz);
        }
        warp_columns(mask, s_col[warp], lane);
        __syncthreads();
        if (tid < SUP_TILES) {
            const uint32_t tx = sx * SUP + (tid & 3), ty = sy * SUP + ((tid >> 2) & 3), tz = sz * SUP + (tid >> 4);
            uint32_t run = 0;
            if (tx < (uint32_t)gx && ty < (uint32_t)gy && tz < (uint32_t)gz) {
                const size_t t = ((size_t)tz * gy + ty) * gx + tx;
                run = tile_incl[t] - tile_count[t] + table2_row(const_cast<uint32_t*>(table2a), const_cast<uint32_t*>(table2b), item, pl1.num_tiles)[tid];
            }
#pragma unroll
            for (int w = 0; w < L2_CHUNK / 32; ++w) {
                s_pre[w][tid] = run;
                run += __popc(s_col[w][tid]);
            }
        }
        __syncthreads();
        while (mask) {
            const int l = __ffsll((long long)mask) - 1;
            mask &= mask - 1;
            point_list[s_pre[warp][l] + __popc(s_col[warp][l] & below)] = g;
        }
    }
}

bool radix_forced() {   // read per call: the parity tests flip it between two forwards of one process
    const char* e = std::getenv("R2X_VOXEL_BINNING");
    return e && std::strcmp(e, "radix") == 0;
}

inline int sup_dim(int g) { return (g + SUP - 1) / SUP; }

}  // namespace

static bool two_level_fits(int gx, int gy, int gz) {
    const long long T = (long long)gx * gy * gz;
    const long long T1 = (long long)sup_dim(gx) * sup_dim(gy) * sup_dim(gz);
    return T > DIRECT_MAX_TILES && T1 <= DIRECT_MAX_TILES;
}

BinPath bin_path(int gx, int gy, int gz, bool has_two_level) {
    if ((long long)gx * gy * gz <= DIRECT_MAX_TILES) return BinPath::Direct;
    return has_two_level && two_level_fits(gx, gy, gz) && !radix_forced() ? BinPath::TwoLevel : BinPath::Radix;
}

size_t two_level_bytes(int P, int gx, int gy, int gz) {
    if (!two_level_fits(gx, gy, gz)) return 0;   // sized by the geometry alone, whatever R2X_VOXEL_BINNING says
    const size_t p = (size_t)(P > 0 ? P : 1);
    const size_t T = (size_t)gx * gy * gz;
    const int T1 = sup_dim(gx) * sup_dim(gy) * sup_dim(gz);
    return align_up(p * 6 * sizeof(uint16_t), 256) + 2 * align_up(p * sizeof(uint32_t), 256) + 256 +
           align_up((size_t)T1 * sizeof(uint2), 256) + plan_bytes(T1) + 256 + directbin_bytes(P, T1) + 256 +
           align_up((size_t)T1 * SUP_TILES * sizeof(uint32_t), 256) + 2 * align_up(T * sizeof(uint32_t), 256) +
           align_up(scan_state_bytes((int)T), 256) + 1024;
}

TwoLevel two_level_view(void* buf, int P, int gx, int gy, int gz, const BinningView& bv) {
    TwoLevel tl;
    const size_t p = (size_t)(P > 0 ? P : 1);
    const size_t T = (size_t)gx * gy * gz;
    tl.gx1 = sup_dim(gx); tl.gy1 = sup_dim(gy); tl.gz1 = sup_dim(gz);
    tl.T1 = tl.gx1 * tl.gy1 * tl.gz1;
    char* q = (char*)align_up((size_t)buf, 256);
    tl.cube1 = (uint16_t*)q; q += align_up(p * 6 * sizeof(uint16_t), 256);
    tl.tiles1 = (uint32_t*)q; q += align_up(p * sizeof(uint32_t), 256);
    tl.offsets1 = (uint32_t*)q; q += align_up(p * sizeof(uint32_t), 256);
    tl.status1 = (uint32_t*)q; q += 256;
    tl.ranges1 = (uint2*)q; q += align_up((size_t)tl.T1 * sizeof(uint2), 256);
    BinningView b1 = bv;
    b1.extra_item = reinterpret_cast<uint2*>(bv.vals[0]);     // level-1 extra items: <= R1 / 256 entries of 8 bytes
    b1.partial = nullptr;
    tl.plan1 = plan_view(q, tl.T1, b1); q += plan_bytes(tl.T1) + 256;
    tl.plan1.chunk_override = L2_CHUNK;
    tl.plan1.max_extra = bv.capacity / 2;
    tl.db1 = directbin_view(q, P, tl.T1); q += directbin_bytes(P, tl.T1) + 256;
    q = (char*)align_up((size_t)q, 256);
    tl.table2a = (uint32_t*)q; q += align_up((size_t)tl.T1 * SUP_TILES * sizeof(uint32_t), 256);
    tl.tile_count = (uint32_t*)q; q += align_up(T * sizeof(uint32_t), 256);
    tl.tile_incl = (uint32_t*)q; q += align_up(T * sizeof(uint32_t), 256);
    tl.scan_state = (void*)q;
    tl.list1 = bv.keys[0];
    tl.table2b = bv.keys[1];
    return tl;
}

int launch_two_level(cudaStream_t st, int P, const uint16_t* cube, const uint32_t* tiles_touched, int gx, int gy, int gz,
                     const uint32_t* status, const TwoLevel& tl, const BinningView& bv, uint2* ranges,
                     const TilePlan& plan) {
    const int T = gx * gy * gz;
    // ---- level 1: Gaussians -> supertiles, with the direct-binning kernels
    super_cube_kernel<<<tl.db1.nb, DIRECT_BLOCK, (size_t)tl.T1 * sizeof(uint32_t), st>>>(P, cube, tiles_touched, tl.cube1,
                                                                                          tl.tiles1, tl.db1, tl.gx1, tl.gy1);
    R2X_CUDA_OK(cudaGetLastError());
    R2X_PASS(launch_direct_scan(st, tl.db1, tl.ranges1, tl.plan1, tl.status1, bv.capacity, nullptr));
    BinningView b1 = bv;
    b1.point_list = tl.list1;
    R2X_PASS(launch_direct_fill(st, P, tl.cube1, tl.tiles1, tl.offsets1, tl.db1, tl.plan1, b1, tl.gx1, tl.gy1,
                                tl.status1));
    // ---- level 2: supertile lists -> tile lists
    int sms;
    R2X_CUDA_OK(sm_count(&sms));
    const int grid = sms * 4;
    fine_count_kernel<<<grid, L2_CHUNK, 0, st>>>(tl.plan1, tl.ranges1, tl.list1, cube, tl.gx1, tl.gy1, tl.table2a,
                                                 tl.table2b, status);
    fine_scan_kernel<<<tl.T1, SUP_TILES, 0, st>>>(tl.plan1, tl.table2a, tl.table2b, tl.gx1, tl.gy1, gx, gy, gz,
                                                  tl.tile_count, status);
    R2X_CUDA_OK(cudaGetLastError());
    R2X_PASS(launch_scan(st, T, tl.tile_count, tl.tile_incl, tl.scan_state, tl.status1 + 2));
    fine_ranges_kernel<<<(T + 255) / 256, 256, 0, st>>>(T, tl.tile_count, tl.tile_incl, status, ranges);
    R2X_CUDA_OK(cudaGetLastError());
    R2X_PASS(launch_plan(st, ranges, plan));
    fine_fill_kernel<<<grid, L2_CHUNK, 0, st>>>(tl.plan1, tl.ranges1, tl.list1, cube, tl.gx1, tl.gy1, gx, gy, gz,
                                                tl.table2a, tl.table2b, tl.tile_count, tl.tile_incl, status,
                                                bv.point_list);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace r2x
