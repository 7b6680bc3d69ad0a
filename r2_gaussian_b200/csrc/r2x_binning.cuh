// r2x_binning.cuh -- tile binning shared by the rasterizer (2-D, 16x16 tiles) and the voxelizer
// (3-D, 8x8x8 tiles): prefix sum over tiles_touched, instance emission, a STABLE least-significant-
// digit radix sort of the instances by tile id only, and per-tile ranges.
//
// Replaces (reference): cub::DeviceScan::InclusiveSum + blocking D2H (RAS/rasterizer_impl.cu:275-279),
// duplicateWithKeys (:70-111), cub::DeviceRadixSort::SortPairs on 64-bit (tile|depth) keys (:298-306),
// identifyTileRanges (:116-138) -- and the 3-D copies in VOX/voxelizer_impl.cu:54-128,244-283.
//
// Design: X-ray accumulation is order-free, so the depth half of the reference key is never sorted on.
// Instances are emitted in the reference's order (Gaussian index ascending, tiles row-major inside the
// bounding rectangle) and moved by a stable sort keyed on the tile id alone (ceil(log2 T) bits ->
// 2 passes of 8 bits for 1024 or 32768 tiles, instead of 6 passes over 64-bit keys).  Stability makes
// every per-tile list ascending in Gaussian index: the render order -- and with it every float sum in
// the forward and backward pass -- is a deterministic function of the inputs.  The reference's
// 64-bit key of an instance is (tile_id << 32) | float_bits(depth[gaussian]); r2x_*_export_keys
// reconstructs it from the sorted list for the bit-exact parity tests.
#pragma once
#include "r2x_common.cuh"

namespace r2x {

struct BinningView {
    // all device pointers, carved out of the caller's binning buffer
    uint32_t* keys[2];     // tile id per instance, ping-pong
    uint32_t* vals[2];     // original instance index, ping-pong
    uint32_t* inst_g;      // [R] Gaussian id of instance i (emission order)
    uint32_t* point_list;  // [R] Gaussian id at sorted position s
    uint32_t* inst_pos;    // [R] emission-order slot of the instance at tile-major position s (backward moments; radix path only)
    uint32_t* hist;        // [256 * SORT_MAX_BLOCKS] digit-major per-block histograms
    uint2* extra_item;     // TilePlan::extra_item
    float* partial;        // TilePlan::partial
    long long capacity;    // instances the buffer can hold
};

constexpr int SORT_THREADS = 256;
constexpr int SORT_ITEMS = 16;                         // keys per thread per sub-chunk
constexpr int SORT_CHUNK = SORT_THREADS * SORT_ITEMS;  // 4096
constexpr int SORT_MAX_BLOCKS = 264;                   // 2 CTAs per SM on the 132 SMs of an H100 SXM

// ---- work plan for the per-tile kernels -------------------------------------------------------
// Per-tile lists are cut into chunks of at most C instances (C = the launch's chunk size, decided ON THE DEVICE by
// plan_chunk_for); a tile of n instances gets ceil(n / C) chunks of EQUAL length (+-1).  A (tile, chunk) pair is one
// work item of the render kernels, handed out through an atomic counter, so that SM load is balanced no matter how
// uneven the per-tile counts are.  Items [0,T) are chunk 0 of every tile (also of empty tiles: they write the
// zeros); items [T, T+E) are the extra chunks, looked up in `extra_item`.  A tile with several chunks combines its
// partial sums in chunk order (the last-arriving CTA does it) => deterministic.
constexpr int PLAN_CHUNK = 256;       // largest chunk = records staged per work item
constexpr int PLAN_MIN_CHUNK = 64;    // smallest chunk (sizes extra_item / partial)
constexpr int PLAN_DONE_SLOTS = 8;   // arrival counters per tile (one per warp of the raster render CTA)
struct TilePlan {
    uint32_t* extra_off;  // [T+1] exclusive scan of (chunks_t - 1); [T] = E
    uint32_t* tile_done;  // [T][PLAN_DONE_SLOTS] arrival counters of multi-chunk tiles
    uint32_t* counter;    // [4]   0: forward queue head, 1: backward queue head, 2: chunk size C of this launch
    uint2* extra_item;    // [R/PLAN_MIN_CHUNK + 1] (tile, chunk >= 1) of extra item j   (binning buffer)
    float* partial;       // [R/PLAN_MIN_CHUNK + 1][512] partial sums of extra chunks      (binning buffer)
    int num_tiles;
    int chunk_override;   // 0 = automatic (plan_chunk_for); else the chunk size to use (two-level binning's level 1)
    int chunk_cap;        // largest chunk the consumer kernels take: PLAN_CHUNK (rasterizer: records staged per item),
                          // VOX_CHUNK_CAP (voxelizer: an item is walked in segments of PLAN_CHUNK records)
    long long max_extra;  // entries in extra_item / partial
};
constexpr int VOX_CHUNK_CAP = 4096;
__host__ __device__ __forceinline__ uint32_t plan_chunk_for(uint32_t R, int chunk_override, int chunk_cap) {
    const uint32_t cap = (uint32_t)(chunk_cap > PLAN_CHUNK ? chunk_cap : PLAN_CHUNK);
    if (chunk_override > 0) return (uint32_t)(chunk_override < PLAN_MIN_CHUNK ? PLAN_MIN_CHUNK : ((uint32_t)chunk_override > cap ? cap : (uint32_t)chunk_override));
    // Rasterizer (cap = PLAN_CHUNK): the largest chunk, because a work item costs the producer warp of the
    // warp-specialised render kernel a fixed latency chain.  Measured (H100 SXM, 400 W, headline scene of 1.06 M
    // instances, render kernel alone): chunks of 256 / 192 / 128 / 64 take 86 / 95 / 104 / 161 us.
    if (cap <= (uint32_t)PLAN_CHUNK) return (uint32_t)PLAN_CHUNK;
    // Voxelizer (cap = VOX_CHUNK_CAP): a tile list is only cut when that is needed to keep a few thousand work items
    // in the queue (64 tiles of a TV crop over the persistent grid: chunks of 256; 32768 tiles of a 256^3 query: one item per tile,
    // so no partial sums leave the CTA and no arrival counters are touched).
    const uint32_t want = (R / 4096u + (uint32_t)PLAN_CHUNK - 1u) / (uint32_t)PLAN_CHUNK * (uint32_t)PLAN_CHUNK;
    return want < (uint32_t)PLAN_CHUNK ? (uint32_t)PLAN_CHUNK : (want > cap ? cap : want);
}
size_t plan_bytes(int num_tiles);
struct BinningView;
TilePlan plan_view(void* image_buf_after_ranges, int num_tiles, const BinningView& bv);
int launch_plan(cudaStream_t st, const uint2* ranges, const TilePlan& plan);
// a forward's plan stays valid for another render of the same lists: rewinds the queue head and the arrival counters
int rewind_plan(cudaStream_t st, const TilePlan& plan);

// Emission-order slot of instance (Gaussian g, tile (tx,ty,tz)): the instances of a Gaussian are contiguous in emission
// order, [offsets[g] - n_g, offsets[g]), tiles of its cube row-major (z, y, x).  Direct binning does not materialise
// the per-instance slot array (it would cost one scattered 4-byte store per instance in the forward, which the
// forward-only users never read); the backward derives the slot from three small per-Gaussian loads instead.
__device__ __forceinline__ uint32_t emission_slot(const uint16_t* __restrict__ cube, const uint32_t* __restrict__ offsets,
                                                  const uint32_t* __restrict__ tiles_touched, uint32_t g, uint32_t tx,
                                                  uint32_t ty, uint32_t tz) {
    const uint32_t* c = reinterpret_cast<const uint32_t*>(cube + 6 * (size_t)g);
    const uint32_t c01 = c[0], c23 = c[1], c45 = c[2];
    const uint32_t x0 = c01 & 0xffff, y0 = c01 >> 16, z0 = c23 & 0xffff, x1 = c23 >> 16, y1 = c45 & 0xffff;
    const uint32_t w = x1 - x0, h = y1 - y0;
    return offsets[g] - tiles_touched[g] + ((tz - z0) * h + (ty - y0)) * w + (tx - x0);
}

// chunk `chunk` of `nch` equal slices of the tile list [r.x, r.y)
__host__ __device__ __forceinline__ void plan_slice(const uint2 r, int chunk, int nch, uint32_t& begin, int& n) {
    // len = q nch + rem: the first `rem` slices hold q + 1 instances, the others q (one 32-bit division)
    const uint32_t len = r.y - r.x;
    const uint32_t q = len / (uint32_t)nch, rem = len - q * (uint32_t)nch;
    const uint32_t c = (uint32_t)chunk;
    begin = r.x + q * c + (c < rem ? c : rem);
    n = (int)(q + (c < rem ? 1u : 0u));
}

__device__ __forceinline__ void plan_decode(const TilePlan& pl, const uint2* __restrict__ ranges, uint32_t item,
                                            int& tile, int& chunk, int& nch, uint32_t& begin, int& n) {
    if ((int)item < pl.num_tiles) { tile = (int)item; chunk = 0; }
    else { const uint2 e = pl.extra_item[item - pl.num_tiles]; tile = (int)e.x; chunk = (int)e.y; }
    nch = (int)(pl.extra_off[tile + 1] - pl.extra_off[tile]) + 1;
    const uint2 r = ranges[tile];
    plan_slice(r, chunk, nch, begin, n);
}

size_t binning_bytes(long long R);
BinningView binning_view(void* buf, long long R);

// ---- which binning a tile grid takes -------------------------------------------------------------
//   Direct    T <= DIRECT_MAX_TILES: per-CTA tile histograms, no instance list, no sort (below)
//   TwoLevel  pipelines that have it (the voxelizer), when the supertile grid fits the direct table (r2x_binning2.cu)
//   Radix     otherwise, or when R2X_VOXEL_BINNING=radix (read per call): emit, stable sort by tile id, ranges
// Only the radix path materialises inst_pos; the others derive emission slots (emission_slot()).
enum class BinPath { Direct, TwoLevel, Radix };
BinPath bin_path(int gx, int gy, int gz, bool has_two_level);

// ---- direct binning (tile counts up to DIRECT_MAX_TILES) ----------------------------------------
// No instance list is materialised and nothing is sorted.  The preprocess CTA b (256 consecutive
// Gaussians) histograms its own instances per tile (`block_tile_histogram`, shared memory) into row b of
// `table`; `direct_scan` does everything that needs grid-wide totals: it turns every tile's column into
// absolute list positions (where CTA b's instances of tile t start in point_list), and publishes the tile
// ranges, the work plan, the CTA instance bases and R; `direct_fill` writes each CTA's Gaussian ids straight
// to their final, stable positions (ascending Gaussian id inside a tile).  4 kernels per forward in total.
constexpr int DIRECT_MAX_TILES = 4096;
constexpr int DIRECT_BLOCK = 256;       // Gaussians per preprocess CTA (== its thread count)
constexpr int DSCAN_COLS = 8;           // tile columns per direct_scan CTA
struct DirectBin {
    uint32_t* table;        // [nb][T]  row b = CTA b's per-tile counts -> absolute list position (direct_scan)
    unsigned long long* lookback;  // [1 + ceil(T / DSCAN_COLS)]  direct_scan's ticket + per-CTA prefix states,
                                   // zeroed by block_tile_histogram
    uint32_t* block_total;  // [nb]  instances of CTA b
    uint32_t* block_base;   // [nb]  exclusive prefix of block_total (direct_scan)
    int num_tiles, nb;
};
__host__ __device__ __forceinline__ int direct_scan_ctas(int num_tiles) { return (num_tiles + DSCAN_COLS - 1) / DSCAN_COLS; }
size_t directbin_bytes(int P, int num_tiles);
DirectBin directbin_view(void* buf, int P, int num_tiles);

// ---- batched views: N views of one cloud binned as one stacked tile grid --------------------------------------------
// View v owns tile rows [v gy, (v + 1) gy) of a gx x N gy grid (a 3-D grid gx x gy x N: the z of a tile is its view) and
// the virtual Gaussians [v Pp, (v + 1) Pp), Pp = P rounded up to DIRECT_BLOCK.  So every direct-binning CTA belongs to
// one view and only counts the band_tiles = gx gy tiles of its band: table is [nb][band_tiles] (db.num_tiles is the
// whole grid's N band_tiles, db.nb = N band_ctas), which keeps the table linear in N.
struct ViewBands {
    int views;        // N
    int band_tiles;   // gx * gy of one view
    int band_ctas;    // Pp / DIRECT_BLOCK
};
size_t directbin_views_bytes(const ViewBands& vb);
DirectBin directbin_views_view(void* buf, const ViewBands& vb);

// Called by all 256 threads of a preprocess CTA.  hist_s: shared uint32[T] scratch, s_wsum: shared uint32[8]
// (the block total's warp sums).  (c01,c23,c45) is the packed tile cube of this thread's Gaussian, n its instance
// count (0 if culled).
__device__ __forceinline__ void block_tile_histogram_into(uint32_t* hist_s, uint32_t* s_wsum, const DirectBin& db,
                                                          uint32_t c01, uint32_t c23, uint32_t c45, uint32_t n, int gx,
                                                          int gy) {
    const int tid = threadIdx.x;
    for (int t = tid; t < db.num_tiles; t += DIRECT_BLOCK) hist_s[t] = 0;
    if (blockIdx.x == 0)   // direct_scan's look-back state (it waits for this grid to finish before reading it)
        for (int i = tid; i <= direct_scan_ctas(db.num_tiles); i += DIRECT_BLOCK) db.lookback[i] = 0ull;
    __syncthreads();
    if (n) {
        const uint32_t x0 = c01 & 0xffff, y0 = c01 >> 16, z0 = c23 & 0xffff, x1 = c23 >> 16, y1 = c45 & 0xffff,
                       z1 = c45 >> 16;
        for (uint32_t z = z0; z < z1; ++z)
            for (uint32_t y = y0; y < y1; ++y) {
                const uint32_t rowb = (z * (uint32_t)gy + y) * (uint32_t)gx;
                for (uint32_t x = x0; x < x1; ++x) atomicAdd(&hist_s[rowb + x], 1u);
            }
    }
    // block total of n (fixed-order tree, result identical for every thread that reads it)
    uint32_t v = n;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0) s_wsum[tid >> 5] = v;
    __syncthreads();
    for (int t = tid; t < db.num_tiles; t += DIRECT_BLOCK) db.table[(size_t)blockIdx.x * db.num_tiles + t] = hist_s[t];
    if (tid == 0) {
        uint32_t tot = 0;
#pragma unroll
        for (int w = 0; w < DIRECT_BLOCK / 32; ++w) tot += s_wsum[w];
        db.block_total[blockIdx.x] = tot;
    }
}
__device__ __forceinline__ void block_tile_histogram(uint32_t* hist_s, const DirectBin& db, uint32_t c01, uint32_t c23,
                                                     uint32_t c45, uint32_t n, int gx, int gy) {
    __shared__ uint32_t s_wsum[DIRECT_BLOCK / 32];
    block_tile_histogram_into(hist_s, s_wsum, db, c01, c23, c45, n, gx, gy);
}

// ---- two-level direct binning (voxel grids with more than DIRECT_MAX_TILES tiles; r2x_binning2.cu) --------------
struct TwoLevel {
    int gx1, gy1, gz1, T1;      // supertile grid (4 x 4 x 4 tiles per supertile)
    uint16_t* cube1;            // [P][6] supertile cube of every Gaussian
    uint32_t* tiles1;           // [P]    supertiles touched
    uint32_t* offsets1;         // [P]    inclusive scan of tiles1 (direct_fill)
    uint32_t* status1;          // [4]    0: R1, 1: level-1 overflow, 2: scratch total of the tile scan
    uint2* ranges1;             // [T1]   supertile lists
    TilePlan plan1;             // level-2 work items = (supertile, chunk of <= 256 entries)
    DirectBin db1;              // level-1 table
    uint32_t* list1;            // [R1]   Gaussian ids, supertile-major, ascending       (binning buffer: keys[0])
    uint32_t* table2a;          // [T1][64]  per-tile counts / prefixes of every supertile's first item
    uint32_t* table2b;          // [E1][64]  ... of the extra items                         (binning buffer: keys[1])
    uint32_t* tile_count;       // [T]
    uint32_t* tile_incl;        // [T]    inclusive scan of tile_count in tile-id order
    void* scan_state;
};
size_t two_level_bytes(int P, int gx, int gy, int gz);   // 0 unless the grid takes two-level binning by its geometry
TwoLevel two_level_view(void* buf, int P, int gx, int gy, int gz, const BinningView& bv);
int launch_two_level(cudaStream_t st, int P, const uint16_t* cube, const uint32_t* tiles_touched, int gx, int gy, int gz,
                     const uint32_t* status, const TwoLevel& tl, const BinningView& bv, uint2* ranges,
                     const TilePlan& plan);

// direct_scan writes ranges[T] and the image-buffer part of the work plan (extra_off, tile_done, counter); the
// extra-item list lives in the binning buffer, which the synchronous variant only allocates once R is known, so
// direct_fill writes it.
int launch_direct_scan(cudaStream_t st, const DirectBin& db, uint2* ranges, const TilePlan& plan, uint32_t* status,
                       long long capacity, uint32_t* status_out);
int launch_direct_fill(cudaStream_t st, int P, const uint16_t* cube, const uint32_t* tiles_touched, uint32_t* offsets,
                       const DirectBin& db, const TilePlan& plan, const BinningView& bv, int gx, int gy,
                       const uint32_t* status);
// the same two stages over the banded table of batched views (P = N Pp virtual Gaussians, gy = one view's tile rows)
int launch_direct_scan_views(cudaStream_t st, const DirectBin& db, const ViewBands& vb, uint2* ranges,
                             const TilePlan& plan, uint32_t* status, long long capacity, uint32_t* status_out);
int launch_direct_fill_views(cudaStream_t st, int P, const uint16_t* cube, const uint32_t* tiles_touched,
                             uint32_t* offsets, const DirectBin& db, const ViewBands& vb, const TilePlan& plan,
                             const BinningView& bv, int gx, int gy, const uint32_t* status);

// Exclusive->inclusive scan of tiles_touched[P] into offsets[P]; total (R) is written to *d_total
// (device) -- single pass, decoupled look-back.  scan_state needs scan_state_bytes(P) bytes, zeroed
// by the call itself.
size_t scan_state_bytes(int P);
int launch_scan(cudaStream_t st, int P, const uint32_t* tiles_touched, uint32_t* offsets, void* scan_state,
                uint32_t* d_total);

// cube: 6 x uint16 per Gaussian (x0,y0,z0,x1,y1,z1); 2-D uses z0=0,z1=1.
int launch_emit(cudaStream_t st, int P, const uint16_t* cube, const uint32_t* tiles_touched,
                const uint32_t* offsets, int gx, int gy, const uint32_t* d_total, const BinningView& bv);

// Stable sort by tile id + per-tile ranges.  `R_launch` sizes the grids (R itself is read on the device
// from d_total so that the same launch sequence works when the host does not know R).
int launch_sort_and_ranges(cudaStream_t st, long long R_launch, int num_tiles, const uint32_t* d_total,
                           const BinningView& bv, uint2* ranges);
// the sort's output: tile id per sorted position (keys[0] or keys[1], by the parity of the pass count)
const uint32_t* sorted_tile_ids(const BinningView& bv, int num_tiles);

// exact 3-NN mean squared distance (r2x_knn.cu)
size_t knn_scratch_bytes(int P);
int launch_knn3(cudaStream_t st, int P, const float* points, float* out, void* scratch, size_t scratch_bytes);

// training-step helpers (r2x_train.cu)
size_t image_loss_scratch_bytes(int H, int W);
int launch_image_loss(cudaStream_t st, int H, int W, const float* image, const float* target, float w_l1,
                      float w_dssim, float* loss_out, float* grad_out, void* scratch, size_t scratch_bytes);
size_t tv3d_scratch_bytes(int nx, int ny, int nz);
int launch_tv3d(cudaStream_t st, int nx, int ny, int nz, const float* vol, int reduction_mean, float* loss_out,
                float* grad_out, void* scratch, size_t scratch_bytes);

}  // namespace r2x
