// r2x_binning.cu -- see r2x_binning.cuh for the design.
#include "r2x_binning.cuh"

namespace r2x {

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

static size_t plan_items(long long R) { return (size_t)(R > 0 ? R : 1) / PLAN_MIN_CHUNK + 1; }

size_t binning_bytes(long long R) {
    size_t r = (size_t)(R > 0 ? R : 1);
    size_t per = align_up(r * sizeof(uint32_t), 256);
    return 7 * per + align_up(256 * SORT_MAX_BLOCKS * sizeof(uint32_t), 256) +
           align_up(plan_items(R) * sizeof(uint2), 256) + align_up(plan_items(R) * 512 * sizeof(float), 256) + 256;
}

BinningView binning_view(void* buf, long long R) {
    BinningView v;
    size_t r = (size_t)(R > 0 ? R : 1);
    size_t per = align_up(r * sizeof(uint32_t), 256);
    char* p = (char*)align_up((size_t)buf, 256);
    v.keys[0] = (uint32_t*)p; p += per;
    v.keys[1] = (uint32_t*)p; p += per;
    v.vals[0] = (uint32_t*)p; p += per;
    v.vals[1] = (uint32_t*)p; p += per;
    v.inst_g = (uint32_t*)p; p += per;
    v.point_list = (uint32_t*)p; p += per;
    v.inst_pos = (uint32_t*)p; p += per;
    v.hist = (uint32_t*)p; p += align_up(256 * SORT_MAX_BLOCKS * sizeof(uint32_t), 256);
    v.extra_item = (uint2*)p; p += align_up(plan_items(R) * sizeof(uint2), 256);
    v.partial = (float*)p;
    v.capacity = R;
    return v;
}

// ------------------------------------------------------------------------------------------------
// Work plan (one CTA; T is at most a few 10^4)
// ------------------------------------------------------------------------------------------------
size_t plan_bytes(int num_tiles) {
    size_t t = (size_t)num_tiles;
    return align_up((t + 1) * sizeof(uint32_t), 256) + align_up(t * PLAN_DONE_SLOTS * sizeof(uint32_t), 256) + 512;
}

TilePlan plan_view(void* buf, int num_tiles, const BinningView& bv) {
    TilePlan pl;
    size_t t = (size_t)num_tiles;
    char* p = (char*)align_up((size_t)buf, 256);
    pl.extra_off = (uint32_t*)p; p += align_up((t + 1) * sizeof(uint32_t), 256);
    pl.tile_done = (uint32_t*)p; p += align_up(t * PLAN_DONE_SLOTS * sizeof(uint32_t), 256);
    pl.counter = (uint32_t*)p;
    pl.extra_item = bv.extra_item;
    pl.partial = bv.partial;
    pl.num_tiles = num_tiles;
    pl.chunk_override = 0;
    pl.chunk_cap = PLAN_CHUNK;
    pl.max_extra = (long long)plan_items(bv.capacity);
    return pl;
}

constexpr int PLAN_RUN = 32;  // consecutive tiles one thread owns per sweep of plan_kernel

// One CTA.  Each thread owns PLAN_RUN consecutive tiles per sweep (1024 * PLAN_RUN tiles), so a
// 256^3 / 8^3 grid (32768 tiles) is one sweep with one CTA-wide scan instead of 32 dependent ones.
__global__ void __launch_bounds__(1024) plan_kernel(const uint2* __restrict__ ranges, TilePlan pl) {
    __shared__ uint32_t s_w[32];
    __shared__ uint32_t s_carry;
    const int T = pl.num_tiles;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // the lists are contiguous and tile-major: the last non-empty tile ends at R
    uint32_t Rloc = 0;
#pragma unroll 4
    for (int t = tid; t < T; t += 1024) Rloc = max(Rloc, ranges[t].y);
    Rloc = __reduce_max_sync(0xffffffffu, Rloc);
    if (tid == 0) s_carry = 0;
    __syncthreads();
    if (lane == 0) atomicMax(&s_carry, Rloc);
    __syncthreads();
    const uint32_t C = plan_chunk_for(s_carry, pl.chunk_override, pl.chunk_cap);
    __syncthreads();
    if (tid == 0) s_carry = 0;
    if (tid < 2) pl.counter[tid] = 0;
    if (tid == 2) pl.counter[2] = C;
    __syncthreads();
    for (int sweep = 0; sweep < T; sweep += 1024 * PLAN_RUN) {
        const int t0 = sweep + tid * PLAN_RUN;
        // extra chunks (beyond the first) of tile t; evaluated twice (sum, then placement) instead of kept in 32 registers
        auto extra_chunks = [&](int t) -> uint32_t {
            if (t >= T) return 0u;
            const uint2 r = ranges[t];
            const uint32_t n = r.y - r.x;
            return n ? (n - 1) / C : 0u;
        };
        uint32_t mine = 0;
#pragma unroll 8
        for (int k = 0; k < PLAN_RUN; ++k) mine += extra_chunks(t0 + k);
        uint32_t incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += up;
        }
        if (lane == 31) s_w[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const uint32_t w = s_w[lane];
            uint32_t x = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t up = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o) x += up;
            }
            s_w[lane] = x - w;
        }
        __syncthreads();
        uint32_t ea = s_carry + s_w[warp] + incl - mine;
#pragma unroll 4
        for (int k = 0; k < PLAN_RUN; ++k) {
            const int t = t0 + k;
            const uint32_t a = extra_chunks(t);
            if (t < T) {
                pl.extra_off[t] = ea;
                for (uint32_t c = 0; c < a; ++c)
                    if ((long long)(ea + c) < pl.max_extra) pl.extra_item[ea + c] = make_uint2((uint32_t)t, c + 1);
            }
            ea += a;
        }
        __syncthreads();
        if (tid == 1023) s_carry = ea;
        __syncthreads();
    }
    if (tid == 0) pl.extra_off[T] = s_carry;
}

int launch_plan(cudaStream_t st, const uint2* ranges, const TilePlan& plan) {
    R2X_CUDA_OK(cudaMemsetAsync(plan.tile_done, 0, sizeof(uint32_t) * (size_t)plan.num_tiles * PLAN_DONE_SLOTS, st));
    plan_kernel<<<1, 1024, 0, st>>>(ranges, plan);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

int rewind_plan(cudaStream_t st, const TilePlan& plan) {
    R2X_CUDA_OK(cudaMemsetAsync(plan.counter, 0, sizeof(uint32_t), st));
    R2X_CUDA_OK(cudaMemsetAsync(plan.tile_done, 0, sizeof(uint32_t) * PLAN_DONE_SLOTS * (size_t)plan.num_tiles, st));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Single-pass inclusive scan (decoupled look-back), 1024 items per CTA.
// state[0] = ticket counter; state[1 + b] = (flag << 62) | value, flag 1 = aggregate, 2 = inclusive.
// ------------------------------------------------------------------------------------------------
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 4;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

size_t scan_state_bytes(int P) { return sizeof(unsigned long long) * (size_t)(2 + (P + SCAN_TILE - 1) / SCAN_TILE); }

__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(int P, const uint32_t* __restrict__ in,
                                                            uint32_t* __restrict__ out,
                                                            unsigned long long* state, uint32_t* d_total,
                                                            int nblocks) {
    __shared__ uint32_t s_bid;
    __shared__ uint32_t s_warp[SCAN_THREADS / 32];
    __shared__ unsigned long long s_excl;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_bid = (uint32_t)atomicAdd(&state[0], 1ull);
    __syncthreads();
    const uint32_t bid = s_bid;
    volatile unsigned long long* st = state + 1;

    const int base = bid * SCAN_TILE + tid * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    if (base + SCAN_ITEMS <= P && ((size_t)(in + base) & 15) == 0) {
        uint4 q = *reinterpret_cast<const uint4*>(in + base);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k) v[k] = (base + k < P) ? in[base + k] : 0u;
    }
    uint32_t tsum = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) { tsum += v[k]; v[k] = tsum; }
    // warp inclusive scan of thread sums
    uint32_t incl = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t wpre = 0, agg = 0;
#pragma unroll
    for (int w = 0; w < SCAN_THREADS / 32; ++w) {
        uint32_t t = s_warp[w];
        if (w < warp) wpre += t;
        agg += t;
    }
    if (tid == 0) {
        unsigned long long excl = 0;
        if (bid == 0) {
            st[0] = (2ull << 62) | (unsigned long long)agg;
        } else {
            st[bid] = (1ull << 62) | (unsigned long long)agg;
            __threadfence();
            int p = (int)bid - 1;
            while (true) {
                unsigned long long s = st[p];
                unsigned long long flag = s >> 62;
                if (flag == 0) continue;
                excl += s & ((1ull << 62) - 1);
                if (flag == 2) break;
                --p;
            }
            st[bid] = (2ull << 62) | (excl + agg);
        }
        __threadfence();
        s_excl = excl;
        if ((int)bid == nblocks - 1) *d_total = (uint32_t)(excl + agg);
    }
    __syncthreads();
    const uint32_t off = (uint32_t)s_excl + wpre + (incl - tsum);
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k)
        if (base + k < P) out[base + k] = off + v[k];
}

int launch_scan(cudaStream_t st, int P, const uint32_t* tiles_touched, uint32_t* offsets, void* scan_state,
                uint32_t* d_total) {
    const int nb = (P + SCAN_TILE - 1) / SCAN_TILE;
    R2X_CUDA_OK(cudaMemsetAsync(scan_state, 0, scan_state_bytes(P), st));
    scan_kernel<<<nb, SCAN_THREADS, 0, st>>>(P, tiles_touched, offsets, (unsigned long long*)scan_state, d_total, nb);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Instance emission: one warp per 32 Gaussians, each covered Gaussian's tiles written by all lanes
// (coalesced).  Order == reference duplicateWithKeys: Gaussian ascending, then z, y, x ascending.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) emit_kernel(int P, const uint16_t* __restrict__ cube,
                                                   const uint32_t* __restrict__ tiles_touched,
                                                   const uint32_t* __restrict__ offsets, int gx, int gy,
                                                   long long capacity, uint32_t* __restrict__ keys,
                                                   uint32_t* __restrict__ inst_g) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    uint32_t n = 0, start = 0, c01 = 0, c23 = 0, c45 = 0;
    if (g < P) {
        n = tiles_touched[g];
        if (n) {
            start = offsets[g] - n;
            const uint32_t* c = reinterpret_cast<const uint32_t*>(cube + 6 * (size_t)g);
            c01 = c[0]; c23 = c[1]; c45 = c[2];
        }
    }
    uint32_t live = __ballot_sync(0xffffffffu, n != 0);
    while (live) {
        const int src = __ffs(live) - 1;
        live &= live - 1;
        const uint32_t n_s = __shfl_sync(0xffffffffu, n, src);
        const uint32_t st_s = __shfl_sync(0xffffffffu, start, src);
        const uint32_t a = __shfl_sync(0xffffffffu, c01, src);
        const uint32_t b = __shfl_sync(0xffffffffu, c23, src);
        const uint32_t c = __shfl_sync(0xffffffffu, c45, src);
        const uint32_t x0 = a & 0xffff, y0 = a >> 16, z0 = b & 0xffff, x1 = b >> 16, y1 = c & 0xffff;
        const uint32_t w = x1 - x0, h = y1 - y0, wh = w * h;
        const uint32_t gid = (uint32_t)(g - lane + src);
        for (uint32_t k = lane; k < n_s; k += 32) {
            const uint32_t z = k / wh, r = k - z * wh, y = r / w, x = r - y * w;
            const uint32_t tile = ((z0 + z) * (uint32_t)gy + (y0 + y)) * (uint32_t)gx + (x0 + x);
            const long long o = (long long)st_s + k;
            if (o < capacity) { keys[o] = tile; inst_g[o] = gid; }
        }
    }
}

int launch_emit(cudaStream_t st, int P, const uint16_t* cube, const uint32_t* tiles_touched,
                const uint32_t* offsets, int gx, int gy, const uint32_t* d_total, const BinningView& bv) {
    (void)d_total;
    if (P <= 0) return 0;
    emit_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, cube, tiles_touched, offsets, gx, gy, bv.capacity, bv.keys[0], bv.inst_g);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Stable LSD radix sort, 8 bits per pass: per-CTA digit histogram -> exclusive scan of the
// digit-major [256 x nb] table -> stable scatter.  Each CTA owns a contiguous range of instances
// (a multiple of SORT_CHUNK) and walks it in order, so order among equal digits is preserved.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ long long per_block_items(long long R, int nb) {
    long long per = (R + nb - 1) / nb;
    return (per + SORT_CHUNK - 1) / SORT_CHUNK * SORT_CHUNK;
}

__global__ void __launch_bounds__(SORT_THREADS) sort_hist_kernel(const uint32_t* __restrict__ keys,
                                                                 const uint32_t* __restrict__ d_total,
                                                                 long long capacity, int shift, int nb,
                                                                 uint32_t* __restrict__ hist) {
    __shared__ uint32_t s_h[256];
    long long R = *d_total;
    if (R > capacity) R = capacity;
    s_h[threadIdx.x] = 0;
    __syncthreads();
    const long long per = per_block_items(R, nb);
    const long long lo = per * blockIdx.x;
    long long hi = lo + per;
    if (hi > R) hi = R;
    for (long long i = lo + threadIdx.x; i < hi; i += SORT_THREADS) atomicAdd(&s_h[(keys[i] >> shift) & 255u], 1u);
    __syncthreads();
    hist[(size_t)threadIdx.x * nb + blockIdx.x] = s_h[threadIdx.x];
}

// exclusive scan of n = 256*nb uint32 in place, one CTA of 1024 threads.  A thread owns SS_RUN consecutive
// entries per sweep: it sums them (independent uint4 loads, one exposed latency), the CTA scans the 1024 sums
// once, and the thread walks its run again (L1/L2 hits) writing the prefixes -- two sweeps for nb = SORT_MAX_BLOCKS.
constexpr int SS_RUN = 64;

__global__ void __launch_bounds__(1024) sort_scan_kernel(uint32_t* __restrict__ hist, int n) {
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024 * SS_RUN) {
        const int i0 = base + tid * SS_RUN;
        const bool whole = i0 + SS_RUN <= n;
        uint32_t sum = 0;
        if (whole) {
#pragma unroll 8
            for (int k = 0; k < SS_RUN; k += 4) {
                const uint4 v = *reinterpret_cast<const uint4*>(hist + i0 + k);
                sum += v.x + v.y + v.z + v.w;
            }
        } else {
            for (int k = 0; k < SS_RUN; ++k)
                if (i0 + k < n) sum += hist[i0 + k];
        }
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const uint32_t w = s_warp[lane];
            uint32_t wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            s_warp[lane] = wi - w;
        }
        __syncthreads();
        uint32_t run = s_carry + s_warp[warp] + incl - sum;
        if (whole) {
#pragma unroll 8
            for (int k = 0; k < SS_RUN; k += 4) {
                const uint4 v = *reinterpret_cast<const uint4*>(hist + i0 + k);
                uint4 o4;
                o4.x = run; run += v.x;
                o4.y = run; run += v.y;
                o4.z = run; run += v.z;
                o4.w = run; run += v.w;
                *reinterpret_cast<uint4*>(hist + i0 + k) = o4;
            }
        } else {
            for (int k = 0; k < SS_RUN; ++k)
                if (i0 + k < n) {
                    const uint32_t v = hist[i0 + k];
                    hist[i0 + k] = run;
                    run += v;
                }
        }
        __syncthreads();
        if (tid == 1023) s_carry = run;
        __syncthreads();
    }
}

template <bool FIRST, bool LAST>
__global__ void __launch_bounds__(SORT_THREADS) sort_scatter_kernel(
    const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in, uint32_t* __restrict__ keys_out,
    uint32_t* __restrict__ vals_out, const uint32_t* __restrict__ inst_g, uint32_t* __restrict__ point_list,
    uint32_t* __restrict__ inst_pos, const uint32_t* __restrict__ d_total, long long capacity, int shift, int nb,
    const uint32_t* __restrict__ hist) {
    constexpr int NW = SORT_THREADS / 32;
    __shared__ uint32_t s_base[256];
    __shared__ uint32_t s_wcnt[NW][256];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long R = *d_total;
    if (R > capacity) R = capacity;
    const long long per = per_block_items(R, nb);
    const long long lo = per * blockIdx.x;
    long long hi = lo + per;
    if (hi > R) hi = R;
    s_base[tid] = hist[(size_t)tid * nb + blockIdx.x];
    const uint32_t lt_mask = (1u << lane) - 1u;

    for (long long cb = lo; cb < hi; cb += SORT_CHUNK) {
#pragma unroll
        for (int w = 0; w < NW; ++w) s_wcnt[w][tid] = 0;
        __syncthreads();
        uint32_t key[SORT_ITEMS];
        uint32_t rnk[SORT_ITEMS];
        const long long wbase = cb + (long long)warp * (32 * SORT_ITEMS);
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; ++k) {
            const long long i = wbase + k * 32 + lane;
            const bool valid = i < hi;
            key[k] = valid ? keys_in[i] : 0u;
            const uint32_t d = valid ? ((key[k] >> shift) & 255u) : 0xffffffffu;
            const uint32_t peers = __match_any_sync(0xffffffffu, d);
            const int leader = __ffs(peers) - 1;
            uint32_t old = 0;
            if (valid && lane == leader) {
                old = s_wcnt[warp][d];
                s_wcnt[warp][d] = old + __popc(peers);
            }
            old = __shfl_sync(0xffffffffu, old, leader);
            rnk[k] = old + __popc(peers & lt_mask);
            __syncwarp();
        }
        __syncthreads();
        {   // per-digit exclusive prefix over warps (thread == digit)
            uint32_t run = 0;
#pragma unroll
            for (int w = 0; w < NW; ++w) {
                const uint32_t t = s_wcnt[w][tid];
                s_wcnt[w][tid] = run;
                run += t;
            }
            __syncthreads();
            // scatter
#pragma unroll
            for (int k = 0; k < SORT_ITEMS; ++k) {
                const long long i = wbase + k * 32 + lane;
                if (i < hi) {
                    const uint32_t d = (key[k] >> shift) & 255u;
                    const uint32_t pos = s_base[d] + s_wcnt[warp][d] + rnk[k];
                    const uint32_t v = FIRST ? (uint32_t)i : vals_in[i];
                    keys_out[pos] = key[k];
                    if (LAST) {
                        point_list[pos] = inst_g[v];
                        inst_pos[pos] = v;
                    } else {
                        vals_out[pos] = v;
                    }
                }
            }
            __syncthreads();
            s_base[tid] += run;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) tile_ranges_kernel(const uint32_t* __restrict__ keys,
                                                          const uint32_t* __restrict__ d_total,
                                                          long long capacity, uint2* __restrict__ ranges) {
    long long R = *d_total;
    if (R > capacity) R = capacity;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < R; i += stride) {
        const uint32_t cur = keys[i];
        if (i == 0) ranges[cur].x = 0;
        else {
            const uint32_t prev = keys[i - 1];
            if (cur != prev) { ranges[prev].y = (uint32_t)i; ranges[cur].x = (uint32_t)i; }
        }
        if (i == R - 1) ranges[cur].y = (uint32_t)R;
    }
}

// ------------------------------------------------------------------------------------------------
// Direct binning
// ------------------------------------------------------------------------------------------------
// table [nb][row_tiles] | look-back [1 + ceil(num_tiles / DSCAN_COLS)] | block_total [nb] | block_base [nb]
static size_t directbin_layout(void* buf, size_t nb, int num_tiles, int row_tiles, DirectBin* db) {
    const size_t t = (size_t)row_tiles;
    const size_t table = align_up(t * nb * sizeof(uint32_t), 256);
    const size_t lookback = align_up((size_t)(1 + direct_scan_ctas(num_tiles)) * sizeof(unsigned long long), 256);
    const size_t per_cta = align_up(nb * sizeof(uint32_t), 256);
    if (db) {
        char* p = (char*)align_up((size_t)buf, 256);
        db->table = (uint32_t*)p; p += table;
        db->lookback = (unsigned long long*)p; p += lookback;
        db->block_total = (uint32_t*)p; p += per_cta;
        db->block_base = (uint32_t*)p;
        db->num_tiles = num_tiles;
        db->nb = (int)nb;
    }
    return table + lookback + 2 * per_cta + 512;
}

static size_t direct_ctas(int P) { return (size_t)((P > 0 ? P : 1) + DIRECT_BLOCK - 1) / DIRECT_BLOCK; }

size_t directbin_bytes(int P, int num_tiles) { return directbin_layout(nullptr, direct_ctas(P), num_tiles, num_tiles, nullptr); }

DirectBin directbin_view(void* buf, int P, int num_tiles) {
    DirectBin db;
    directbin_layout(buf, direct_ctas(P), num_tiles, num_tiles, &db);
    return db;
}

size_t directbin_views_bytes(const ViewBands& vb) {
    return directbin_layout(nullptr, (size_t)vb.views * vb.band_ctas, vb.views * vb.band_tiles, vb.band_tiles, nullptr);
}

DirectBin directbin_views_view(void* buf, const ViewBands& vb) {
    DirectBin db;
    directbin_layout(buf, (size_t)vb.views * vb.band_ctas, vb.views * vb.band_tiles, vb.band_tiles, &db);
    return db;
}

// direct_scan: CTA k (in ticket order) owns the DSCAN_COLS tile columns [8k, 8k + 8) of table[nb][T].  Thread
// (seg, col) sums a run of consecutive rows of one column (a warp reads 4 rows x 32 bytes, whole sectors); the run
// sums are scanned over the segments, which gives every tile's total and every row's prefix inside the column.  The
// tile starts -- an exclusive scan of the tile totals in tile order -- and the extra-chunk offsets of the work plan
// come from a decoupled look-back over the CTAs in ticket order (one 64-bit state per CTA: flag | extra chunks |
// instances).  The column is then rewritten as absolute list positions, ranges[t].x + prefix[b][t], and the CTA
// publishes ranges, extra_off and the zeroed arrival counters of its tiles.  Every CTA also reduces block_total,
// so R, the overflow flag and the chunk size C are known before any tile start is; CTA 0 writes block_base,
// status and the queue counters.  The kernel is a chain of dependent round trips (ticket, loads, look-back, stores);
// small CTAs run it fastest (H100 at 700 W, headline scene: 5.5 / 6.2 / 8.1 us with 256 / 512 / 1024 threads).
constexpr int DSCAN_THREADS = 256;
constexpr int DSCAN_WARPS = DSCAN_THREADS / 32;
constexpr int DSCAN_SEGS = DSCAN_THREADS / DSCAN_COLS;   // 32 row segments
constexpr int DSCAN_KEEP = 16;                           // rows of a segment kept in registers between the passes
static_assert(DSCAN_COLS == 8, "a warp is 4 row segments x 8 columns");
constexpr unsigned long long LB_AGG = 1ull << 62, LB_INCL = 2ull << 62, LB_VALUE = (1ull << 62) - 1;

// VIEWS = true (batched views): the column of tile t is made of the band_ctas rows of its view's CTAs, rows
// band_tiles long (ViewBands); all other rows are zero for t and are neither stored nor read.
template <bool VIEWS>
__device__ __forceinline__ void direct_scan_body(DirectBin db, ViewBands vb, uint2* __restrict__ ranges, TilePlan pl,
                                                 uint32_t* __restrict__ status, long long capacity,
                                                 uint32_t* __restrict__ status_out) {
    pdl_prologue();
    __shared__ uint32_t s_w[DSCAN_WARPS];
    __shared__ uint32_t s_wcol[DSCAN_WARPS][DSCAN_COLS];
    __shared__ uint32_t s_tot[DSCAN_COLS];
    __shared__ uint32_t s_bid;
    __shared__ unsigned long long s_excl;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int T = db.num_tiles, nb = db.nb, nctas = gridDim.x;
    if (tid == 0) s_bid = (uint32_t)atomicAdd(&db.lookback[0], 1ull);

    // ---- R = sum of the CTA instance totals (every CTA); CTA 0 also writes their exclusive prefix, block_base
    const int K = (nb + DSCAN_THREADS - 1) / DSCAN_THREADS;
    uint32_t mine = 0;
    for (int k = 0; k < K; ++k) {
        const int i = tid * K + k;
        if (i < nb) mine += db.block_total[i];
    }
    uint32_t incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t x = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += x;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t R = 0, wpre = 0;
#pragma unroll 8
    for (int w = 0; w < DSCAN_WARPS; ++w) {
        const uint32_t x = s_w[w];
        wpre += (w < warp) ? x : 0u;
        R += x;
    }
    const bool ov = (long long)R > capacity;
    const uint32_t C = plan_chunk_for(R, pl.chunk_override, pl.chunk_cap);
    if (blockIdx.x == 0) {
        uint32_t run = wpre + incl - mine;
        for (int k = 0; k < K; ++k) {
            const int i = tid * K + k;
            if (i < nb) {
                const uint32_t v = db.block_total[i];
                db.block_base[i] = run;
                run += v;
            }
        }
        if (tid == 0) {
            status[0] = R;
            status[1] = ov ? 1u : 0u;
            if (status_out) { status_out[0] = R; status_out[1] = ov ? 1u : 0u; }
            pl.counter[0] = pl.counter[1] = pl.counter[3] = 0;
            pl.counter[2] = C;
        }
    }

    // ---- column sums
    const int bid = (int)s_bid;
    const int col = tid & (DSCAN_COLS - 1), seg = tid / DSCAN_COLS;
    const int t = bid * DSCAN_COLS + col;
    int rows = nb, stride = T;
    uint32_t* cp = db.table + t;
    if constexpr (VIEWS) {
        const int v = t / vb.band_tiles;
        rows = vb.band_ctas;
        stride = vb.band_tiles;
        cp = db.table + (size_t)v * vb.band_ctas * vb.band_tiles + (t - v * vb.band_tiles);
    }
    const int rps = (rows + DSCAN_SEGS - 1) / DSCAN_SEGS;
    const int r0 = min(seg * rps, rows), r1 = min(r0 + rps, rows);
    const bool live = t < T;
    uint32_t keep[DSCAN_KEEP];
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < DSCAN_KEEP; ++k) {
        keep[k] = (live && r0 + k < r1) ? cp[(size_t)(r0 + k) * stride] : 0u;
        sum += keep[k];
    }
    if (live)
        for (int r = r0 + DSCAN_KEEP; r < r1; ++r) sum += cp[(size_t)r * stride];
    // prefix over the segments: 4 segments per warp (lanes 8 apart), then over the warps
    uint32_t sincl = sum;
#pragma unroll
    for (int o = DSCAN_COLS; o < 32; o <<= 1) {
        const uint32_t x = __shfl_up_sync(0xffffffffu, sincl, o);
        if (lane >= o) sincl += x;
    }
    if (lane >= 32 - DSCAN_COLS) s_wcol[warp][col] = sincl;
    __syncthreads();
    uint32_t pre = sincl - sum, tot = 0;
#pragma unroll 8
    for (int w = 0; w < DSCAN_WARPS; ++w) {
        const uint32_t x = s_wcol[w][col];
        pre += (w < warp) ? x : 0u;
        tot += x;
    }
    if (tid < DSCAN_COLS) s_tot[tid] = tot;   // warp 0: tot of column tid
    __syncthreads();
    // the CTA's tiles in order: instances and extra chunks before column `col`, and in all 8 columns
    uint32_t cnt_before = 0, ext_before = 0, cnt_all = 0, ext_all = 0;
#pragma unroll
    for (int c = 0; c < DSCAN_COLS; ++c) {
        const uint32_t n = s_tot[c];
        const uint32_t e = n ? (n - 1) / C : 0u;
        cnt_before += (c < col) ? n : 0u;
        ext_before += (c < col) ? e : 0u;
        cnt_all += n;
        ext_all += e;
    }

    // ---- decoupled look-back over the CTAs in ticket order, one warp, 32 predecessors per probe
    if (warp == 0) {
        volatile unsigned long long* st = db.lookback + 1;
        const unsigned long long agg = ((unsigned long long)ext_all << 32) | cnt_all;
        unsigned long long excl = 0;
        if (bid == 0) {
            if (lane == 0) st[0] = LB_INCL | agg;
        } else {
            if (lane == 0) st[bid] = LB_AGG | agg;
            int top = bid - 1;
            while (true) {
                const int q = top - lane;
                const unsigned long long s = q >= 0 ? (unsigned long long)st[q] : LB_INCL;
                const uint32_t incl_lanes = __ballot_sync(0xffffffffu, (s >> 62) == 2ull);
                const uint32_t wait_lanes = __ballot_sync(0xffffffffu, (s >> 62) == 0ull);
                const int stop = incl_lanes ? __ffs(incl_lanes) - 1 : 31;   // nearest inclusive state
                const uint32_t upto = stop == 31 ? 0xffffffffu : ((2u << stop) - 1u);
                if (wait_lanes & upto) continue;                          // a predecessor has not published yet
                unsigned long long v = (lane <= stop) ? (s & LB_VALUE) : 0ull;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                excl += v;
                if (incl_lanes) break;
                top -= 32;
            }
            if (lane == 0) st[bid] = LB_INCL | (excl + agg);
        }
        if (lane == 0) s_excl = excl;
    }
    __syncthreads();
    const uint32_t start = (uint32_t)s_excl + cnt_before;              // first list position of tile t
    const uint32_t eoff = (uint32_t)(s_excl >> 32) + ext_before;       // its first extra work item
    if (live) {
        uint32_t pos = start + pre;
#pragma unroll
        for (int k = 0; k < DSCAN_KEEP; ++k)
            if (r0 + k < r1) {
                cp[(size_t)(r0 + k) * stride] = pos;
                pos += keep[k];
            }
        for (int r = r0 + DSCAN_KEEP; r < r1; ++r) {
            const uint32_t a = cp[(size_t)r * stride];
            cp[(size_t)r * stride] = pos;
            pos += a;
        }
        // Overflow (asynchronous variant only): the binning buffer cannot hold the lists, so EMPTY ranges are
        // published -- the render then produces zeros without touching unwritten list entries -- and the host sees
        // status[1] = 1 and re-runs with a larger buffer.
        if (seg == 0) {
            ranges[t] = ov ? make_uint2(0u, 0u) : make_uint2(start, start + tot);
            pl.extra_off[t] = ov ? 0u : eoff;
        }
    }
    if (tid < DSCAN_COLS * PLAN_DONE_SLOTS) {
        const size_t i = (size_t)bid * DSCAN_COLS * PLAN_DONE_SLOTS + tid;
        if (i < (size_t)T * PLAN_DONE_SLOTS) pl.tile_done[i] = 0;
    }
    if (bid == nctas - 1 && tid == 0) pl.extra_off[T] = ov ? 0u : (uint32_t)(s_excl >> 32) + ext_all;
}

__global__ void __launch_bounds__(DSCAN_THREADS) direct_scan_kernel(DirectBin db, uint2* __restrict__ ranges, TilePlan pl,
                                                                    uint32_t* __restrict__ status, long long capacity,
                                                                    uint32_t* __restrict__ status_out) {
    direct_scan_body<false>(db, ViewBands{1, db.num_tiles, db.nb}, ranges, pl, status, capacity, status_out);
}

__global__ void __launch_bounds__(DSCAN_THREADS) direct_scan_views_kernel(DirectBin db, ViewBands vb,
                                                                          uint2* __restrict__ ranges, TilePlan pl,
                                                                          uint32_t* __restrict__ status,
                                                                          long long capacity,
                                                                          uint32_t* __restrict__ status_out) {
    direct_scan_body<true>(db, vb, ranges, pl, status, capacity, status_out);
}

int launch_direct_scan(cudaStream_t st, const DirectBin& db, uint2* ranges, const TilePlan& plan, uint32_t* status,
                       long long capacity, uint32_t* status_out) {
    R2X_CUDA_OK(pdl_launch(direct_scan_kernel, dim3(direct_scan_ctas(db.num_tiles)), dim3(DSCAN_THREADS), 0, st, db,
                           ranges, plan, status, capacity, status_out));
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_direct_scan_views(cudaStream_t st, const DirectBin& db, const ViewBands& vb, uint2* ranges,
                             const TilePlan& plan, uint32_t* status, long long capacity, uint32_t* status_out) {
    R2X_CUDA_OK(pdl_launch(direct_scan_views_kernel, dim3(direct_scan_ctas(db.num_tiles)), dim3(DSCAN_THREADS), 0, st, db,
                           vb, ranges, plan, status, capacity, status_out));
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// CTA b places the instances of Gaussians [256 b, 256 b + 256).  It marks, per tile, WHICH of its Gaussians touch
// the tile (a 256-bit mask per tile, word w = warp w's 32 Gaussians, one ATOMS.OR per instance), turns the word
// populations into per-word ranks, and then every thread walks the tiles of ITS OWN Gaussian again (lane per instance,
// the same loop as the marking); the instance goes to
//     table[b][t] (direct_scan: where CTA b's run of tile t starts in point_list)
//       + rank of the Gaussian among the CTA's Gaussians on tile t = wrank[w][t] + popc(mask[w][t] & lanes below)
// => every tile list is ascending in Gaussian id (the stable order) without any search, sort or warp match, and the
// instance's emission-order slot (backward moments) follows from offsets[] (emission_slot(), r2x_binning.cuh).
// Written one by one, the ids would be one scattered 4-byte store each, and those stores are what the kernel's time
// goes to.  So when the CTA's instances fit `stage_cap`, they are first put in shared memory in (tile, rank) order --
// the order of their positions inside each run -- and then stored with consecutive threads on consecutive entries, so
// a warp's store covers whole runs.  The CTA also writes the extra-item list of the work plan for its slice of the
// tiles (the list lives in the binning buffer; see launch_direct_scan).
// Dynamic shared memory: mask[8][T] u32 | base[T] u32 | wrank[8][T] u8 | (staged:) loc[T] u32 | pos[cap] u32 | id[cap] u8
// (the Gaussian's index inside the CTA).
constexpr int FILL_STAGE_TILES = 4 * DIRECT_BLOCK;   // staging when T <= 1024 ...
constexpr int FILL_STAGE_CAP = 4608;                 // ... for up to 4608 instances per CTA: 70.5 KB, 3 CTAs per SM

// VIEWS = true (batched views): CTA b belongs to one view, its table row and its shared tables cover that view's band
// (T = band_tiles, tiles numbered band-locally: the tile cube's z, the view, is dropped); the work plan's extra items
// cover the whole grid (T_all = db.num_tiles).
template <bool VIEWS>
__device__ __forceinline__ void direct_fill_body(int P, const uint16_t* __restrict__ cube,
                                                 const uint32_t* __restrict__ tiles_touched,
                                                 uint32_t* __restrict__ offsets, DirectBin db, TilePlan pl,
                                                 uint32_t* __restrict__ point_list, int gx, int gy,
                                                 const uint32_t* __restrict__ status, int stage_cap, int band_tiles) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ uint32_t s_w8[8];
    __shared__ uint32_t s_ct[4][8];
    const int T = VIEWS ? band_tiles : db.num_tiles;
    const int T_all = db.num_tiles;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t* s_mask = reinterpret_cast<uint32_t*>(smem_raw);                    // [8][T]
    uint32_t* s_base = s_mask + 8 * (size_t)T;                                    // [T]
    unsigned char* s_wrank = reinterpret_cast<unsigned char*>(s_base + T);        // [8][T]
    uint32_t* s_loc = reinterpret_cast<uint32_t*>(s_wrank + 8 * (size_t)T);      // [T]
    uint32_t* s_pos = s_loc + T;                                                  // [stage_cap]
    unsigned char* s_id = reinterpret_cast<unsigned char*>(s_pos + stage_cap);   // [stage_cap]
    // shared memory only: done while direct_scan may still be running
    for (int i = tid; i < 2 * T; i += DIRECT_BLOCK) reinterpret_cast<uint4*>(s_mask)[i] = make_uint4(0u, 0u, 0u, 0u);
    pdl_prologue();

    const int b = blockIdx.x;
    const int g = b * DIRECT_BLOCK + tid;
    uint32_t n = 0, c01 = 0, c23 = 0, c45 = 0;
    if (g < P) {
        n = tiles_touched[g];
        const uint32_t* c = reinterpret_cast<const uint32_t*>(cube + 6 * (size_t)g);
        c01 = c[0]; c23 = c[1]; c45 = c[2];
    }
    const uint32_t bbase = db.block_base[b];   // instance base of this CTA (direct_scan)
    const bool ov = status[1] != 0u;           // overflow (direct_scan): nothing may be written to point_list
    const uint32_t* row = db.table + (size_t)b * T;   // rewritten by direct_scan even on overflow
    for (int t = tid; t < T; t += DIRECT_BLOCK) s_base[t] = row[t];
    // CTA-exclusive scan of n
    uint32_t ia = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t x = __shfl_up_sync(0xffffffffu, ia, o);
        if (lane >= o) ia += x;
    }
    if (lane == 31) s_w8[warp] = ia;
    __syncthreads();
    uint32_t wpre = 0, total = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        const uint32_t x = s_w8[w];
        wpre += (w < warp) ? x : 0u;
        total += x;
    }
    if (g < P) offsets[g] = bbase + wpre + ia;    // inclusive scan, same meaning as the reference's point_offsets
    if (ov) return;                                // uniform across the grid
    // extra work items of the tiles [b K, b K + K): (tile, chunk >= 1)
    {
        const int K = (T_all + (int)gridDim.x - 1) / (int)gridDim.x;
        const int t1 = min(T_all, (b + 1) * K);
        for (int t = b * K + tid; t < t1; t += DIRECT_BLOCK) {
            const uint32_t eo = pl.extra_off[t], ne = pl.extra_off[t + 1] - eo;
            for (uint32_t c = 0; c < ne; ++c)
                if ((long long)(eo + c) < pl.max_extra) pl.extra_item[eo + c] = make_uint2((uint32_t)t, c + 1);
        }
    }
    const uint32_t x0 = c01 & 0xffff, y0 = c01 >> 16, x1 = c23 >> 16, y1 = c45 & 0xffff;
    const uint32_t z0 = VIEWS ? 0u : (c23 & 0xffff), z1 = VIEWS ? 1u : (c45 >> 16);
    // mark
    {
        uint32_t* plane = s_mask + (size_t)warp * T;
        const uint32_t bit = 1u << lane;
        if (n)
            for (uint32_t z = z0; z < z1; ++z)
                for (uint32_t y = y0; y < y1; ++y) {
                    const uint32_t rowb = (z * (uint32_t)gy + y) * (uint32_t)gx;
                    for (uint32_t x = x0; x < x1; ++x) atomicOr(&plane[rowb + x], bit);
                }
    }
    __syncthreads();
    // rank of word w inside its tile's run = population of the words below it; returns the CTA's count on tile t
    auto word_ranks = [&](int t) -> uint32_t {
        uint32_t run = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            s_wrank[(size_t)w * T + t] = (unsigned char)run;    // <= 224
            run += __popc(s_mask[(size_t)w * T + t]);
        }
        return run;
    };
    const bool staged = stage_cap > 0 && total <= (uint32_t)stage_cap;   // uniform; stage_cap > 0 only when T <= 1024
    if (staged) {
        // loc[t] = where tile t's run starts in the staging buffer: exclusive scan of the counts in tile order
        // (tile t = k * 256 + tid: K <= 4 interleaved scans at once)
        uint32_t cnt[4], inc[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int t = k * DIRECT_BLOCK + tid;
            cnt[k] = t < T ? word_ranks(t) : 0u;
            inc[k] = cnt[k];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t x = __shfl_up_sync(0xffffffffu, inc[k], o);
                if (lane >= o) inc[k] += x;
            }
            if (lane == 31) s_ct[k][warp] = inc[k];
        }
        __syncthreads();
        uint32_t carry = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            uint32_t before = 0, all = 0;
#pragma unroll
            for (int w = 0; w < 8; ++w) {
                const uint32_t x = s_ct[k][w];
                before += (w < warp) ? x : 0u;
                all += x;
            }
            const int t = k * DIRECT_BLOCK + tid;
            if (t < T) s_loc[t] = carry + before + inc[k] - cnt[k];
            carry += all;
        }
    } else {
        for (int t = tid; t < T; t += DIRECT_BLOCK) word_ranks(t);
    }
    __syncthreads();
    // place: lane per instance, tiles of this thread's Gaussian in emission order (z, y, x ascending)
    if (n) {
        const uint32_t* plane = s_mask + (size_t)warp * T;
        const unsigned char* wr = s_wrank + (size_t)warp * T;
        const uint32_t below = (1u << lane) - 1u;
        for (uint32_t z = z0; z < z1; ++z)
            for (uint32_t y = y0; y < y1; ++y) {
                const uint32_t rowb = (z * (uint32_t)gy + y) * (uint32_t)gx;
                for (uint32_t x = x0; x < x1; ++x) {
                    const uint32_t t = rowb + x;
                    const uint32_t r = wr[t] + __popc(plane[t] & below);
                    if (staged) {
                        const uint32_t slot = s_loc[t] + r;
                        s_pos[slot] = s_base[t] + r;
                        s_id[slot] = (unsigned char)tid;
                    } else {
                        point_list[s_base[t] + r] = (uint32_t)g;
                    }
                }
            }
    }
    if (staged) {
        __syncthreads();
        const uint32_t g0 = (uint32_t)b * DIRECT_BLOCK;
        for (uint32_t i = tid; i < total; i += DIRECT_BLOCK) point_list[s_pos[i]] = g0 + s_id[i];
    }
}

__global__ void __launch_bounds__(DIRECT_BLOCK) direct_fill_kernel(int P, const uint16_t* __restrict__ cube,
                                                                   const uint32_t* __restrict__ tiles_touched,
                                                                   uint32_t* __restrict__ offsets, DirectBin db,
                                                                   TilePlan pl, uint32_t* __restrict__ point_list,
                                                                   int gx, int gy, const uint32_t* __restrict__ status,
                                                                   int stage_cap) {
    direct_fill_body<false>(P, cube, tiles_touched, offsets, db, pl, point_list, gx, gy, status, stage_cap, 0);
}

__global__ void __launch_bounds__(DIRECT_BLOCK) direct_fill_views_kernel(
    int P, const uint16_t* __restrict__ cube, const uint32_t* __restrict__ tiles_touched, uint32_t* __restrict__ offsets,
    DirectBin db, TilePlan pl, uint32_t* __restrict__ point_list, int gx, int gy, const uint32_t* __restrict__ status,
    int stage_cap, int band_tiles) {
    direct_fill_body<true>(P, cube, tiles_touched, offsets, db, pl, point_list, gx, gy, status, stage_cap, band_tiles);
}

int launch_direct_fill_views(cudaStream_t st, int P, const uint16_t* cube, const uint32_t* tiles_touched,
                             uint32_t* offsets, const DirectBin& db, const ViewBands& vb, const TilePlan& plan,
                             const BinningView& bv, int gx, int gy, const uint32_t* status) {
    const int T = vb.band_tiles;   // a CTA's shared tables cover its view's band
    const int cap = T <= FILL_STAGE_TILES ? FILL_STAGE_CAP : 0;
    const size_t smem = (size_t)T * (cap ? 48 : 44) + (size_t)cap * 5;
    if (smem > 48 * 1024)
        R2X_CUDA_OK(cudaFuncSetAttribute(direct_fill_views_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         DIRECT_MAX_TILES * 44));
    R2X_CUDA_OK(pdl_launch(direct_fill_views_kernel, dim3(db.nb), dim3(DIRECT_BLOCK), smem, st, P, cube, tiles_touched,
                           offsets, db, plan, bv.point_list, gx, gy, status, cap, T));
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_direct_fill(cudaStream_t st, int P, const uint16_t* cube, const uint32_t* tiles_touched, uint32_t* offsets,
                       const DirectBin& db, const TilePlan& plan, const BinningView& bv, int gx, int gy,
                       const uint32_t* status) {
    static_assert(FILL_STAGE_TILES <= 4 * DIRECT_BLOCK, "the staging scan handles at most 4 tiles per thread");
    static_assert(FILL_STAGE_TILES * 48 + FILL_STAGE_CAP * 5 <= DIRECT_MAX_TILES * 44, "one attribute covers both layouts");
    const int T = db.num_tiles;
    const int cap = T <= FILL_STAGE_TILES ? FILL_STAGE_CAP : 0;
    const size_t smem = (size_t)T * (cap ? 48 : 44) + (size_t)cap * 5;
    if (smem > 48 * 1024)
        R2X_CUDA_OK(cudaFuncSetAttribute(direct_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         DIRECT_MAX_TILES * 44));
    R2X_CUDA_OK(pdl_launch(direct_fill_kernel, dim3(db.nb), dim3(DIRECT_BLOCK), smem, st, P, cube, tiles_touched, offsets,
                           db, plan, bv.point_list, gx, gy, status, cap));
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// 8-bit passes over the ceil(log2 T) bits of a tile id
static int sort_passes(int num_tiles) {
    int bits = 1;
    while ((1ll << bits) < (long long)num_tiles) ++bits;
    return (bits + 7) / 8;
}

const uint32_t* sorted_tile_ids(const BinningView& bv, int num_tiles) { return bv.keys[sort_passes(num_tiles) & 1]; }

int launch_sort_and_ranges(cudaStream_t st, long long R_launch, int num_tiles, const uint32_t* d_total,
                           const BinningView& bv, uint2* ranges) {
    R2X_CUDA_OK(cudaMemsetAsync(ranges, 0, sizeof(uint2) * (size_t)num_tiles, st));
    if (R_launch <= 0) return 0;
    const int passes = sort_passes(num_tiles);
    long long nbl = (R_launch + SORT_CHUNK - 1) / SORT_CHUNK;
    const int nb = (int)(nbl < SORT_MAX_BLOCKS ? nbl : SORT_MAX_BLOCKS);
    int cur = 0;
    for (int p = 0; p < passes; ++p) {
        const int shift = 8 * p;
        const bool first = (p == 0), last = (p == passes - 1);
        sort_hist_kernel<<<nb, SORT_THREADS, 0, st>>>(bv.keys[cur], d_total, bv.capacity, shift, nb, bv.hist);
        sort_scan_kernel<<<1, 1024, 0, st>>>(bv.hist, 256 * nb);
#define R2X_SCATTER(F, L)                                                                                          \
    sort_scatter_kernel<F, L><<<nb, SORT_THREADS, 0, st>>>(bv.keys[cur], bv.vals[cur], bv.keys[cur ^ 1],           \
                                                           bv.vals[cur ^ 1], bv.inst_g, bv.point_list, bv.inst_pos, \
                                                           d_total, bv.capacity, shift, nb, bv.hist)
        if (first && last) R2X_SCATTER(true, true);
        else if (first) R2X_SCATTER(true, false);
        else if (last) R2X_SCATTER(false, true);
        else R2X_SCATTER(false, false);
#undef R2X_SCATTER
        R2X_CUDA_OK(cudaGetLastError());
        cur ^= 1;
    }
    long long nbr = (R_launch + 255) / 256;
    int sms;
    R2X_CUDA_OK(sm_count(&sms));
    const int gr = (int)(nbr < sms * 8 ? nbr : sms * 8);
    tile_ranges_kernel<<<gr, 256, 0, st>>>(bv.keys[cur], d_total, bv.capacity, ranges);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace r2x
