// ball_query.cuh -- block-level building blocks of the index-exact ball query (shared by grouping.cu and sa_train.cu).
//
// Reference semantics (pointnet2/tf_ops/grouping/tf_grouping_g.cu:3-36): for every query scan the dataset in index
// order, keep the first `nsample` points with max(sqrtf(d2),1e-20f) < radius, fill the unused slots with the first hit,
// report the (clamped) count.  "First nsample in index order" == "the nsample smallest indices among ALL in-radius
// points", which is what lets a spatial grid in:
//
//   grid path   the CTA bins its cloud (already staged in shared memory) into cells of size 1.001*radius (at most 16 per
//               axis) with a counting sort; a query only tests the points of its 3x3x3 cell neighbourhood (~5 % of a
//               uniform cloud instead of 100 %), compacts the hits with ballots, ranks them by index (counting rank) and
//               emits the nsample smallest in ascending order -- bit-identical output, ~3x fewer instructions;
//   scan path   the ordered brute-force scan (128 points per warp step, early exit), used when the cloud or the query has a
//               non-finite coordinate (a NaN distance counts as inside in the reference), when the grid would be
//               degenerate, when the cloud does not fit the grid's shared-memory budget, or when a query collects more
//               than kBqHitCap hits (dense neighbourhoods: exactly where the early-exit scan is fast).
// The distance test is the same arithmetic in both paths: d2 = fma(dz,dz,fma(dx,dx,dy*dy)) and !(d2 > T) with T the largest
// float whose sqrtf is < radius (see grouping.cu).
#pragma once
#include "common.cuh"

namespace psa {

constexpr int kBqWarps = 8;
constexpr int kBqThreads = kBqWarps * 32;
constexpr int kBqGridMax = 16;          // cells per axis
constexpr int kBqMaxCells = kBqGridMax * kBqGridMax * kBqGridMax;
constexpr int kBqHitCap = 128;          // in-radius candidates a query may collect on the grid path
constexpr int kBqGridMaxN = 4096;       // clouds larger than this use the scan path only (shared-memory budget)

struct BqGrid {
    float minx, miny, minz, inv_h;
    int gx, gy, gz;
    int use;                            // 0 -> scan path for the whole CTA
};

// Shared-memory plan.  scan mode: the cloud as SoA (12 B/point).  grid mode: ONLY the cell-sorted copy (16 B/point) + cell
// table + hit buffers -- the rare scan fallback then reads the cloud from global memory / L1 -- so that four CTAs fit an SM.
struct BqSmem {
    float* sx; float* sy; float* sz;    // scan mode: np = round_up(n,128) floats each, padded with +inf; grid mode: null
    float4* sorted;                     // grid mode: n entries (x, y, z, bits(k)), grouped by cell
    int* cell_end;                      // grid mode: kBqMaxCells + 32 ints: end offset of each cell, scratch
    int* hits;                          // grid mode: kBqWarps * bq_warp_scratch_words(n)
    const float* gxyz;                  // the cloud in global memory (AoS), always valid
    unsigned short* pos_of;             // optional (grid mode): pos_of[k] = slot of point k in `sorted`; null = not kept
};

constexpr int kBqSlabQueries = 8;      // queries a warp searches at a time on the lane-per-slab path (3 lanes each)
__host__ __device__ inline int bq_bitmap_words_per_lane(int n) { return ((n + 31) / 32 + 31) / 32; }   // a query's bitmap = 32 * this words
// per-warp scratch in grid mode: the hit list of the warp-per-query search or the 8 bitmaps of the lane-per-slab search
__host__ __device__ inline int bq_warp_scratch_words(int n) {
    const int bm = kBqSlabQueries * 32 * bq_bitmap_words_per_lane(n);
    return bm > kBqHitCap ? bm : kBqHitCap;
}
__host__ __device__ inline size_t bq_smem_bytes(int n, bool grid) {
    if (grid) return (size_t)n * 16 + (size_t)(kBqMaxCells + 32) * 4 + (size_t)kBqWarps * bq_warp_scratch_words(n) * 4;
    return (size_t)((n + 127) & ~127) * 3 * sizeof(float);
}
__host__ __device__ inline bool bq_grid_fits(int n) { return n <= kBqGridMaxN; }

__device__ __forceinline__ BqSmem bq_carve(float* base, int n, bool grid, const float* gxyz) {
    BqSmem s;
    s.gxyz = gxyz;
    s.pos_of = nullptr;
    if (grid) {
        s.sx = s.sy = s.sz = nullptr;
        s.sorted = reinterpret_cast<float4*>(base);
        s.cell_end = reinterpret_cast<int*>(s.sorted + n);
        s.hits = s.cell_end + kBqMaxCells + 32;
    } else {
        const int np = (n + 127) & ~127;
        s.sx = base; s.sy = base + np; s.sz = base + 2 * np;
        s.sorted = nullptr; s.cell_end = nullptr; s.hits = nullptr;
    }
    return s;
}

__device__ __forceinline__ int bq_cell_coord(float v, float vmin, float inv_h, int g) {
    const int c = (int)((v - vmin) * inv_h);
    return c < g - 1 ? c : g - 1;
}

// scan mode: stage the cloud (AoS global -> SoA shared, padded with +inf).
// grid mode: each thread keeps its points (k = tid + 256 i) in registers, the CTA computes the bounding box, bins the
// points with a counting sort and scatters (x, y, z, k) into `sorted`.  All kBqThreads call.
template <int PPT>   // points per thread in grid mode: n <= PPT * kBqThreads
__device__ __forceinline__ BqGrid bq_stage_and_build(const BqSmem& s, int n, float radius, bool want_grid) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* p1 = s.gxyz;
    const float inf = __int_as_float(0x7f800000);
    BqGrid g;
    g.use = 0; g.minx = g.miny = g.minz = 0.f; g.inv_h = 0.f; g.gx = g.gy = g.gz = 1;
    if (!want_grid) {
        const int np = (n + 127) & ~127;
        const int total = n * 3;
        int i = tid;
        for (; i + 7 * kBqThreads < total; i += 8 * kBqThreads) {
            float v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = __ldg(p1 + i + u * kBqThreads);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int e = i + u * kBqThreads, k = e / 3, c = e - k * 3;
                (c == 0 ? s.sx : (c == 1 ? s.sy : s.sz))[k] = v[u];
            }
        }
        for (; i < total; i += kBqThreads) {
            const int k = i / 3, c = i - k * 3;
            (c == 0 ? s.sx : (c == 1 ? s.sy : s.sz))[k] = __ldg(p1 + i);
        }
        for (int k = n + tid; k < np; k += kBqThreads) { s.sx[k] = inf; s.sy[k] = inf; s.sz[k] = inf; }
        __syncthreads();
        return g;
    }
    float px[PPT], py[PPT], pz[PPT];
    float mnx = inf, mny = inf, mnz = inf, mxx = -inf, mxy = -inf, mxz = -inf;
    bool fin = true;
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
        const int k = tid + i * kBqThreads;
        if (k < n) {
            px[i] = __ldg(p1 + 3 * k); py[i] = __ldg(p1 + 3 * k + 1); pz[i] = __ldg(p1 + 3 * k + 2);
            fin = fin && fabsf(px[i]) <= 3.0e38f && fabsf(py[i]) <= 3.0e38f && fabsf(pz[i]) <= 3.0e38f;
            mnx = fminf(mnx, px[i]); mny = fminf(mny, py[i]); mnz = fminf(mnz, pz[i]);
            mxx = fmaxf(mxx, px[i]); mxy = fmaxf(mxy, py[i]); mxz = fmaxf(mxz, pz[i]);
        } else {
            px[i] = py[i] = pz[i] = 0.f;
        }
    }
    // ---- bounding box + finiteness: warp shuffles, then 8 partials through shared memory ----
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mnx = fminf(mnx, __shfl_xor_sync(0xffffffffu, mnx, o)); mny = fminf(mny, __shfl_xor_sync(0xffffffffu, mny, o));
        mnz = fminf(mnz, __shfl_xor_sync(0xffffffffu, mnz, o)); mxx = fmaxf(mxx, __shfl_xor_sync(0xffffffffu, mxx, o));
        mxy = fmaxf(mxy, __shfl_xor_sync(0xffffffffu, mxy, o)); mxz = fmaxf(mxz, __shfl_xor_sync(0xffffffffu, mxz, o));
    }
    fin = __all_sync(0xffffffffu, fin);
    float* scratch = reinterpret_cast<float*>(s.cell_end);
    if (lane == 0) {
        scratch[warp * 8 + 0] = mnx; scratch[warp * 8 + 1] = mny; scratch[warp * 8 + 2] = mnz;
        scratch[warp * 8 + 3] = mxx; scratch[warp * 8 + 4] = mxy; scratch[warp * 8 + 5] = mxz;
        scratch[warp * 8 + 6] = fin ? 1.f : 0.f;
    }
    __syncthreads();
    {
        float bmn[3] = {inf, inf, inf}, bmx[3] = {-inf, -inf, -inf};
        bool bfin = true;
#pragma unroll
        for (int w = 0; w < kBqWarps; ++w) {
#pragma unroll
            for (int c = 0; c < 3; ++c) { bmn[c] = fminf(bmn[c], scratch[w * 8 + c]); bmx[c] = fmaxf(bmx[c], scratch[w * 8 + 3 + c]); }
            bfin = bfin && scratch[w * 8 + 6] != 0.f;
        }
        const float rx = bmx[0] - bmn[0], ry = bmx[1] - bmn[1], rz = bmx[2] - bmn[2];
        const float rmax = fmaxf(rx, fmaxf(ry, rz));
        const float h = fmaxf(radius * 1.001f, rmax * (1.0f / kBqGridMax) * 1.001f);   // cell >= 1.001 r, <= 16 cells per axis
        g.minx = bmn[0]; g.miny = bmn[1]; g.minz = bmn[2];
        g.inv_h = 1.0f / h;
        g.gx = min(kBqGridMax, (int)(rx * g.inv_h) + 1);
        g.gy = min(kBqGridMax, (int)(ry * g.inv_h) + 1);
        g.gz = min(kBqGridMax, (int)(rz * g.inv_h) + 1);
        // a grid of fewer than 27 cells prunes nothing; non-finite coordinates need the reference's NaN semantics
        g.use = (bfin && n >= 1 && h > 0.f && h <= 3.0e38f && g.gx * g.gy * g.gz >= 27) ? 1 : 0;
    }
    __syncthreads();                     // scratch (cell_end) is about to be reused
    if (!g.use) return g;
    const int ncells = g.gx * g.gy * g.gz;
    for (int c = tid; c < ncells; c += kBqThreads) s.cell_end[c] = 0;
    __syncthreads();
    int cell[PPT];
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
        const int k = tid + i * kBqThreads;
        cell[i] = 0;
        if (k < n) {
            const int cx = bq_cell_coord(px[i], g.minx, g.inv_h, g.gx), cy = bq_cell_coord(py[i], g.miny, g.inv_h, g.gy);
            const int cz = bq_cell_coord(pz[i], g.minz, g.inv_h, g.gz);
            cell[i] = (cz * g.gy + cy) * g.gx + cx;
            atomicAdd(&s.cell_end[cell[i]], 1);
        }
    }
    __syncthreads();
    // exclusive scan of the cell counts: each thread owns a contiguous run of cells
    {
        const int per = (ncells + kBqThreads - 1) / kBqThreads;      // <= 16
        const int c0 = tid * per;
        int local = 0;
        for (int c = c0; c < min(ncells, c0 + per); ++c) local += s.cell_end[c];
        int incl = local;                                            // warp inclusive scan
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        int* wsum = s.cell_end + kBqMaxCells;                        // 8 warp totals
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        int off = incl - local;
        for (int w = 0; w < warp; ++w) off += wsum[w];
        for (int c = c0; c < min(ncells, c0 + per); ++c) { const int cnt = s.cell_end[c]; s.cell_end[c] = off; off += cnt; }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
        const int k = tid + i * kBqThreads;
        if (k < n) {
            const int pos = atomicAdd(&s.cell_end[cell[i]], 1);      // afterwards cell_end[c] = END of cell c
            s.sorted[pos] = make_float4(px[i], py[i], pz[i], __int_as_float(k));
            if (s.pos_of != nullptr) s.pos_of[k] = (unsigned short)pos;
        }
    }
    __syncthreads();
    return g;
}

// squared distances of two dataset points to one query, as float pairs: per element the reference's
// FMUL(dy*dy), FFMA(dx,dx), FFMA(dz,dz) (x_k - q instead of q - x_k: identical squares)
__device__ __forceinline__ float2 bq_dist2_pair(float2 x, float2 y, float2 z, float2 nqx, float2 nqy, float2 nqz) {
    const float2 dx = fadd2_rn(x, nqx), dy = fadd2_rn(y, nqy), dz = fadd2_rn(z, nqz);
    float2 t = fmul2_rn(dy, dy);
    t = ffma2_rn(dx, dx, t);
    t = ffma2_rn(dz, dz, t);
    return t;
}

// Ordered scan path: one warp, 128 points per step (4 consecutive points per lane), ballot + prefix-popcount compaction
// keeps index order, early exit.  The points come from the shared SoA copy (scan mode) or, in grid mode where this is
// only the rare fallback, straight from global memory.
__device__ __forceinline__ int bq_scan_warp(int n, int nsample, float thr, bool none, const BqSmem& s, float qx, float qy,
                                            float qz, int* idxrow, int lane) {
    int cnt = 0, first = -1;
    if (!none) {
        const float2 nqx = make_float2(-qx, -qx), nqy = make_float2(-qy, -qy), nqz = make_float2(-qz, -qz);
        const unsigned lt = lanemask_lt();
        const float inf = __int_as_float(0x7f800000);
        for (int base = 0; base < n && cnt < nsample; base += 128) {
            const int k = base + lane * 4;
            float4 X, Y, Z;
            if (s.sx != nullptr) {
                X = *reinterpret_cast<const float4*>(s.sx + k);
                Y = *reinterpret_cast<const float4*>(s.sy + k);
                Z = *reinterpret_cast<const float4*>(s.sz + k);
            } else {
                float v[12];
#pragma unroll
                for (int u = 0; u < 12; ++u) v[u] = (k + u / 3 < n) ? __ldg(s.gxyz + (size_t)k * 3 + u) : inf;
                X = make_float4(v[0], v[3], v[6], v[9]); Y = make_float4(v[1], v[4], v[7], v[10]); Z = make_float4(v[2], v[5], v[8], v[11]);
            }
            const float2 d01 = bq_dist2_pair(make_float2(X.x, X.y), make_float2(Y.x, Y.y), make_float2(Z.x, Z.y), nqx, nqy, nqz);
            const float2 d23 = bq_dist2_pair(make_float2(X.z, X.w), make_float2(Y.z, Y.w), make_float2(Z.z, Z.w), nqx, nqy, nqz);
            // !(d > thr): a NaN distance counts as inside, exactly like the reference's max(sqrtf(NaN),1e-20f) < r
            bool i0 = !(d01.x > thr), i1 = !(d01.y > thr), i2 = !(d23.x > thr), i3 = !(d23.y > thr);
            if (base + 128 > n) {   // last chunk: the +inf padding must not count even when the QUERY is NaN
                i0 = i0 && (k < n); i1 = i1 && (k + 1 < n); i2 = i2 && (k + 2 < n); i3 = i3 && (k + 3 < n);
            }
            const unsigned m4 = (i0 ? 1u : 0u) | (i1 ? 2u : 0u) | (i2 ? 4u : 0u) | (i3 ? 8u : 0u);
            const unsigned anyb = __ballot_sync(0xffffffffu, m4 != 0u);
            if (anyb == 0u) continue;
            const unsigned b0 = __ballot_sync(0xffffffffu, i0), b1 = __ballot_sync(0xffffffffu, i1);
            const unsigned b2 = __ballot_sync(0xffffffffu, i2), b3 = __ballot_sync(0xffffffffu, i3);
            if (first < 0) {
                const int lf = __ffs(anyb) - 1;
                const unsigned mf = __shfl_sync(0xffffffffu, m4, lf);
                first = base + lf * 4 + (__ffs(mf) - 1);
            }
            int pos = cnt + __popc(b0 & lt) + __popc(b1 & lt) + __popc(b2 & lt) + __popc(b3 & lt);
            if (i0) { if (pos < nsample) idxrow[pos] = k; ++pos; }
            if (i1) { if (pos < nsample) idxrow[pos] = k + 1; ++pos; }
            if (i2) { if (pos < nsample) idxrow[pos] = k + 2; ++pos; }
            if (i3) { if (pos < nsample) idxrow[pos] = k + 3; }
            cnt += __popc(b0) + __popc(b1) + __popc(b2) + __popc(b3);
        }
    }
    if (cnt > nsample) cnt = nsample;
    const int fillv = first < 0 ? 0 : first;
    for (int l = cnt + lane; l < nsample; l += 32) idxrow[l] = fillv;   // tf_grouping_g.cu:26-29
    return cnt;
}

// One warp, one query.  Writes the idx row (global or shared memory) and returns the clamped count.
__device__ __forceinline__ int bq_query_warp(int n, int nsample, float thr, bool none, const BqSmem& s, const BqGrid& g,
                                             float qx, float qy, float qz, int* idxrow, int lane, int warp) {
    const bool qfin = fabsf(qx) <= 3.0e38f && fabsf(qy) <= 3.0e38f && fabsf(qz) <= 3.0e38f;
    if (!g.use || !qfin || none) return bq_scan_warp(n, nsample, thr, none, s, qx, qy, qz, idxrow, lane);
    // ---- the (up to) nine x-contiguous cell runs of the 3x3x3 neighbourhood, one per lane 0..8 ----
    const float fx = fminf(fmaxf((qx - g.minx) * g.inv_h, -2.f), (float)(kBqGridMax + 1));
    const float fy = fminf(fmaxf((qy - g.miny) * g.inv_h, -2.f), (float)(kBqGridMax + 1));
    const float fz = fminf(fmaxf((qz - g.minz) * g.inv_h, -2.f), (float)(kBqGridMax + 1));
    const int cqx = (int)floorf(fx), cqy = (int)floorf(fy), cqz = (int)floorf(fz);
    const int lox = max(cqx - 1, 0), hix = min(cqx + 1, g.gx - 1);
    int start = 0, len = 0;
    if (lane < 9 && lox <= hix) {
        const int cy = cqy + (lane % 3) - 1, cz = cqz + (lane / 3) - 1;
        if (cy >= 0 && cy < g.gy && cz >= 0 && cz < g.gz) {
            const int rb = (cz * g.gy + cy) * g.gx;
            start = (rb + lox == 0) ? 0 : s.cell_end[rb + lox - 1];
            len = s.cell_end[rb + hix] - start;
        }
    }
    int incl = len;
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 8);
    int r_start[9], r_end[9];          // candidate slot t belongs to run i iff r_end[i-1] <= t < r_end[i]
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        r_start[i] = __shfl_sync(0xffffffffu, start, i);
        r_end[i] = __shfl_sync(0xffffffffu, incl, i);
    }
    // ---- test the candidates, compact the hits (any order) ----
    int* hits = s.hits + warp * bq_warp_scratch_words(n);
    const unsigned lt = lanemask_lt();
    int nh = 0;
    for (int t0 = 0; t0 < total; t0 += 32) {
        const int t = t0 + lane;
        bool in = false;
        int k = 0;
        if (t < total) {
            int sel = r_start[0] + t;
#pragma unroll
            for (int i = 1; i < 9; ++i)
                if (t >= r_end[i - 1]) sel = r_start[i] + (t - r_end[i - 1]);
            const float4 p = s.sorted[sel];
            k = __float_as_int(p.w);
            in = !(dist2_ref_gpu(qx - p.x, qy - p.y, qz - p.z) > thr);
        }
        const unsigned b = __ballot_sync(0xffffffffu, in);
        if (in) { const int pos = nh + __popc(b & lt); if (pos < kBqHitCap) hits[pos] = k; }
        nh += __popc(b);
        if (nh > kBqHitCap) break;       // warp-uniform
    }
    __syncwarp();
    if (nh > kBqHitCap) return bq_scan_warp(n, nsample, thr, none, s, qx, qy, qz, idxrow, lane);
    // ---- rank the hits by index: the reference keeps the nsample smallest, in ascending order ----
    int first = 0x7fffffff;
    for (int h0 = 0; h0 < nh; h0 += 32) {
        const int h = h0 + lane;
        const int mine = h < nh ? hits[h] : 0x7fffffff;
        int rank = 0;
        for (int j = 0; j < nh; ++j) rank += (hits[j] < mine) ? 1 : 0;     // broadcast reads; indices are distinct
        if (h < nh && rank < nsample) idxrow[rank] = mine;
        first = min(first, mine);
    }
    first = __reduce_min_sync(0xffffffffu, first);
    const int cnt = min(nh, nsample);
    const int fillv = nh > 0 ? first : 0;
    for (int l = cnt + lane; l < nsample; l += 32) idxrow[l] = fillv;
    return cnt;
}

// ---------------------------------------------------------------------------------------------------------------------
// Lane-per-slab search (used by the streaming F1 kernel and ball_query_kernel v3).
//
// The warp-per-query search above spends most of its instructions on warp-uniform bookkeeping (run table, slot -> run
// selection, ranking): ~600 warp instructions per query.  Here THREE lanes own a query: lane t walks the three x-runs of
// the z-slab cqz + t - 1 of the 3x3x3 cell neighbourhood point by point and sets bit k of the query's bitmap (n bits in
// shared memory) for every in-radius point k.  The reference's "first nsample in index order" is then the nsample lowest
// set bits -- read out by the whole warp (bq_extract_bitmap) in ascending order with popcount prefix sums, independent of
// how many points are inside the ball (no hit cap, no ranking).  Same distance arithmetic, same cell geometry (cells
// >= 1.001 r), so the set of hits is the one the scan finds: index-exact.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kBqSlabLanes = 3;


// One lane, one z-slab (t = 0,1,2) of the neighbourhood of a FINITE query on a usable grid.
__device__ __forceinline__ void bq_search_slab(const BqSmem& s, const BqGrid& g, float thr, float qx, float qy, float qz, int t,
                                               unsigned* __restrict__ bitmap) {
    const float fx = fminf(fmaxf((qx - g.minx) * g.inv_h, -2.f), (float)(kBqGridMax + 1));
    const float fy = fminf(fmaxf((qy - g.miny) * g.inv_h, -2.f), (float)(kBqGridMax + 1));
    const float fz = fminf(fmaxf((qz - g.minz) * g.inv_h, -2.f), (float)(kBqGridMax + 1));
    const int cqx = (int)floorf(fx), cqy = (int)floorf(fy), cz = (int)floorf(fz) + t - 1;
    const int lox = max(cqx - 1, 0), hix = min(cqx + 1, g.gx - 1);
    if (lox > hix || cz < 0 || cz >= g.gz) return;
#pragma unroll 1
    for (int dy = -1; dy <= 1; ++dy) {
        const int cy = cqy + dy;
        if (cy < 0 || cy >= g.gy) continue;
        const int rb = (cz * g.gy + cy) * g.gx;
        int p = (rb + lox == 0) ? 0 : s.cell_end[rb + lox - 1];
        const int e = s.cell_end[rb + hix];
        // two candidates per trip: the second load is clamped into the run and masked
        for (; p < e; p += 2) {
            const float4 a = s.sorted[p];
            const float4 b = s.sorted[min(p + 1, e - 1)];
            const bool ia = !(dist2_ref_gpu(qx - a.x, qy - a.y, qz - a.z) > thr);
            const bool ib = !(dist2_ref_gpu(qx - b.x, qy - b.y, qz - b.z) > thr) && (p + 1 < e);
            if (ia) { const int k = __float_as_int(a.w); atomicOr(bitmap + (k >> 5), 1u << (k & 31)); }
            if (ib) { const int k = __float_as_int(b.w); atomicOr(bitmap + (k >> 5), 1u << (k & 31)); }
        }
    }
}

// Whole warp: the nsample lowest set bits of `bitmap` (32 * wpl words, lane l owns words [l*wpl, (l+1)*wpl)) in ascending
// order -> idxrow[0..cnt), remaining slots filled with the first hit (0 if none: tf_grouping_g.cu:26-29); clears the bitmap.
__device__ __forceinline__ int bq_extract_bitmap(unsigned* __restrict__ bitmap, int wpl, int nsample, int* __restrict__ idxrow, int lane) {
    unsigned w[4];
    int c = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        w[i] = 0u;
        if (i < wpl) { w[i] = bitmap[lane * wpl + i]; bitmap[lane * wpl + i] = 0u; c += __popc(w[i]); }
    }
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    const unsigned have = __ballot_sync(0xffffffffu, c > 0);
    int firstbit = 0;
#pragma unroll
    for (int i = 3; i >= 0; --i)
        if (w[i] != 0u) firstbit = (lane * wpl + i) * 32 + __ffs(w[i]) - 1;
    const int first = have ? __shfl_sync(0xffffffffu, firstbit, __ffs(have) - 1) : 0;
    int pos = incl - c;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        unsigned x = w[i];
        while (x != 0u && pos < nsample) {
            const int bit = __ffs(x) - 1;
            x &= x - 1u;
            idxrow[pos++] = (lane * wpl + i) * 32 + bit;
        }
    }
    const int cnt = min(total, nsample);
    for (int l = cnt + lane; l < nsample; l += 32) idxrow[l] = first;
    return cnt;
}

// LPQ lanes per query, 32/LPQ queries per warp at once: the nsample lowest set bits of a bitmap of LPQ*WPS words (lane `sub`
// of the group owns words [sub*WPS, (sub+1)*WPS), read ONCE into registers) in ascending order -> idxrow[0..cnt), rest filled
// with the first hit (0 if none).  Every lane of the warp must call (shuffles); groups with active == false do nothing else.
template <int LPQ, int WPS>
__device__ __forceinline__ int bq_extract_bitmap_sub(const unsigned* __restrict__ bitmap, int nsample, int* __restrict__ idxrow, int lane, bool active) {
    const int sub = lane & (LPQ - 1);
    unsigned w[WPS];
    int c = 0;
#pragma unroll
    for (int i = 0; i < WPS; ++i) {
        w[i] = active ? bitmap[sub * WPS + i] : 0u;
        c += __popc(w[i]);
    }
    int incl = c;
#pragma unroll
    for (int o = 1; o < LPQ; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o, LPQ);
        if (sub >= o) incl += v;
    }
    const int total = __shfl_sync(0xffffffffu, incl, LPQ - 1, LPQ);
    const unsigned have = (__ballot_sync(0xffffffffu, c > 0) >> (lane & (32 - LPQ))) & (LPQ == 32 ? 0xffffffffu : ((1u << (LPQ & 31)) - 1u));
    int firstbit = 0;
#pragma unroll
    for (int i = WPS - 1; i >= 0; --i)
        if (w[i] != 0u) firstbit = (sub * WPS + i) * 32 + __ffs(w[i]) - 1;
    const int first = __shfl_sync(0xffffffffu, firstbit, have ? __ffs(have) - 1 : 0, LPQ);
    if (!active) return 0;
    int pos = incl - c;
#pragma unroll
    for (int i = 0; i < WPS; ++i) {
        unsigned x = w[i];
        while (x != 0u && pos < nsample) {
            const int bit = __ffs(x) - 1;
            x &= x - 1u;
            idxrow[pos++] = (sub * WPS + i) * 32 + bit;
        }
    }
    const int cnt = min(total, nsample);
    const int fillv = have ? first : 0;
    for (int l = cnt + sub; l < nsample; l += LPQ) idxrow[l] = fillv;
    return cnt;
}

}  // namespace psa
