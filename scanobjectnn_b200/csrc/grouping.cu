// grouping.cu -- ball query, group_point (+grad), SelectionSort / knn_point for sm_90a.
//
// Replaces pointnet2/tf_ops/grouping/tf_grouping_g.cu of the reference (one CTA per cloud, one thread per
// query walking all n points from global memory).  The ball query itself lives in ball_query.cuh (spatial grid +
// ordered-scan fallback, index-exact).  Here: the cloud's coordinates are staged once per CTA in
// shared memory as SoA, one WARP owns a query and tests 32 consecutive points per step, and the reference's
// "first nsample in index order" rule is kept by ballot + prefix-popcount compaction, tiles consumed in
// ascending order, with a per-query early exit.  The sqrt of the reference's `max(sqrtf(d2),1e-20f) < r` test
// is hoisted to the host: sqrtf is monotone, so the test equals `!(d2 > T)` with T the largest float whose
// correctly-rounded sqrt is < r (NaN d2 counts as inside, exactly like CUDA's max(NaN,1e-20f) = 1e-20f < r).
#include <math.h>
#include <string.h>

#include "ball_query.cuh"
#include "common.cuh"

namespace psa {

// Largest t >= 0 with sqrtf(t) < r, or `none` when no distance can satisfy max(sqrtf(d2),1e-20f) < r.
float ball_query_threshold(float radius, bool* none) {
    *none = !(radius > 1e-20f);   // also catches NaN
    if (*none) return 0.f;
    uint32_t lo = 0u, hi = 0x7f7fffffu;   // sqrtf(+0) = 0 < r holds
    while (lo < hi) {
        uint32_t mid = lo + (hi - lo + 1u) / 2u;
        float t;
        memcpy(&t, &mid, 4);
        if (sqrtf(t) < radius) lo = mid; else hi = mid - 1u;
    }
    float t;
    memcpy(&t, &lo, 4);
    return t;
}

template <int PPT>
__global__ void __launch_bounds__(kBqThreads, PPT <= 8 ? 3 : 2)
ball_query_kernel(int n, int m, int nsample, float radius, float thr, int none, int want_grid, int q_per_cta,
                  const float* __restrict__ xyz1, const float* __restrict__ xyz2, int* __restrict__ idx,
                  int* __restrict__ pts_cnt) {
    extern __shared__ __align__(16) float smem_f[];
    const int cloud = blockIdx.y;
    const BqSmem s = bq_carve(smem_f, n, want_grid != 0, xyz1 + (size_t)cloud * n * 3);
    const BqGrid g = bq_stage_and_build<PPT>(s, n, radius, want_grid != 0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int q0 = blockIdx.x * q_per_cta;
    const int q1 = min(m, q0 + q_per_cta);
    const float* p2 = xyz2 + (size_t)cloud * m * 3;
    if (g.use && !none) {
        // lane-per-slab search: three lanes per query, eight queries per warp step, hits as bits of a per-query bitmap, the
        // nsample lowest bits read out in order (ball_query.cuh); non-finite queries take the ordered scan
        const int wpl = bq_bitmap_words_per_lane(n);
        unsigned* bm = reinterpret_cast<unsigned*>(s.hits) + (size_t)warp * bq_warp_scratch_words(n);
        for (int i = lane; i < kBqSlabQueries * 32 * wpl; i += 32) bm[i] = 0u;
        __syncwarp();
        const int qi = lane / kBqSlabLanes, tsl = lane - qi * kBqSlabLanes;
        for (int q = q0 + warp * kBqSlabQueries; q < q1; q += kBqWarps * kBqSlabQueries) {
            const int nq = min(kBqSlabQueries, q1 - q);
            float qx = 0.f, qy = 0.f, qz = 0.f;
            if (qi < nq) { qx = __ldg(p2 + (q + qi) * 3 + 0); qy = __ldg(p2 + (q + qi) * 3 + 1); qz = __ldg(p2 + (q + qi) * 3 + 2); }
            const bool qfin = fabsf(qx) <= 3.0e38f && fabsf(qy) <= 3.0e38f && fabsf(qz) <= 3.0e38f;
            if (qi < nq && qfin) bq_search_slab(s, g, thr, qx, qy, qz, tsl, bm + (size_t)qi * 32 * wpl);
            __syncwarp();
            for (int i = 0; i < nq; ++i) {
                const bool fin_i = __shfl_sync(0xffffffffu, qfin ? 1 : 0, i * kBqSlabLanes) != 0;
                int* row = idx + ((size_t)cloud * m + q + i) * nsample;
                int cnt;
                if (fin_i) {
                    cnt = bq_extract_bitmap(bm + (size_t)i * 32 * wpl, wpl, nsample, row, lane);
                } else {
                    const float cx = __shfl_sync(0xffffffffu, qx, i * kBqSlabLanes), cy = __shfl_sync(0xffffffffu, qy, i * kBqSlabLanes);
                    const float cz = __shfl_sync(0xffffffffu, qz, i * kBqSlabLanes);
                    cnt = bq_scan_warp(n, nsample, thr, false, s, cx, cy, cz, row, lane);
                }
                if (pts_cnt != nullptr && lane == 0) pts_cnt[(size_t)cloud * m + q + i] = cnt;
            }
            __syncwarp();
        }
        return;
    }
    for (int q = q0 + warp; q < q1; q += kBqWarps) {
        const float qx = __ldg(p2 + q * 3 + 0), qy = __ldg(p2 + q * 3 + 1), qz = __ldg(p2 + q * 3 + 2);
        int* row = idx + ((size_t)cloud * m + q) * nsample;
        const int cnt = bq_scan_warp(n, nsample, thr, none != 0, s, qx, qy, qz, row, lane);
        if (pts_cnt != nullptr && lane == 0) pts_cnt[(size_t)cloud * m + q] = cnt;
    }
}

// out[b,j,k,:] = points[b, idx[b,j,k], :]
template <typename VT>
__global__ void group_point_kernel(int n, int cv, long long rows_per_b, long long total, const VT* __restrict__ points,
                                   const int* __restrict__ idx, VT* __restrict__ out) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        long long row = e / cv;
        int l = (int)(e - row * cv);
        long long bi = row / rows_per_b;
        int ii = __ldg(idx + row);
        out[e] = __ldg(points + (bi * n + ii) * cv + l);
    }
}

// ---- SelectionSort (tf_grouping_g.cu:83-123): one warp per (b,j) row, row resident in shared memory ----
// Round s: position of the FIRST strict minimum in [s,n) (the reference starts min=s and scans t>s with '<',
// so the earliest position among equal minima wins), swap with slot s carrying indices.
__device__ __forceinline__ void selection_rounds(int n, int k, float* v, int* id, int lane) {
    for (int s = 0; s < k && s < n; ++s) {
        // every lane starts from the reference's `min = s`; a NaN at s can never be displaced (x < NaN is false)
        float best = v[s];
        int bpos = s;
        for (int t = s + 1 + lane; t < n; t += 32) {
            float x = v[t];
            if (x < best) { best = x; bpos = t; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            float ob = __shfl_xor_sync(0xffffffffu, best, o);
            int op = __shfl_xor_sync(0xffffffffu, bpos, o);
            if (ob < best || (ob == best && op < bpos)) { best = ob; bpos = op; }
        }
        if (lane == 0 && bpos != s) {
            float tv = v[bpos]; v[bpos] = v[s]; v[s] = tv;
            int ti = id[bpos]; id[bpos] = id[s]; id[s] = ti;
        }
        __syncwarp();
    }
}

constexpr int kSelWarps = 4;

__global__ void __launch_bounds__(kSelWarps * 32)
selection_sort_kernel(long long rows, int n, int k, const float* __restrict__ dist, int* __restrict__ outi,
                      float* __restrict__ out) {
    extern __shared__ float smem_f[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* v = smem_f + (size_t)warp * n * 2;
    int* id = reinterpret_cast<int*>(v + n);
    for (long long r = (long long)blockIdx.x * kSelWarps + warp; r < rows; r += (long long)gridDim.x * kSelWarps) {
        const float* d = dist + r * n;
        for (int t = lane; t < n; t += 32) { v[t] = d[t]; id[t] = t; }
        __syncwarp();
        selection_rounds(n, k, v, id, lane);
        for (int t = lane; t < n; t += 32) { out[r * n + t] = v[t]; outi[r * n + t] = id[t]; }
        __syncwarp();
    }
}

// One streaming pass over a row of distances keeps the k smallest (value, index) sorted, one per lane (k <= 32), and the
// smallest value that did NOT make the list (rejected on arrival or evicted later) = the (k+1)-th smallest of the row.
// If the k list values are pairwise distinct and the k-th is strictly below that runner-up, the selection sort's result
// does not depend on its swaps -- it IS this list -- and it is written; any tie (duplicate points), NaN or unfilled slot
// returns false and the exact swap-by-swap rounds decide, as in the reference.  `dist(t)` = this lane's candidate t < n.
template <class DistFn>
__device__ __forceinline__ bool knn_fast_path(int n, int k, DistFn dist, int lane, float* __restrict__ val_out, int* __restrict__ idx_out) {
    const float inf = __int_as_float(0x7f800000);
    float lv = inf, thr_v = inf;
    int li = 0x7fffffff, thr_i = 0x7fffffff;
    float rej = inf;                  // per lane: smallest candidate this lane saw rejected; lane-uniform part folded in below
    float ev = inf;                   // uniform: smallest value evicted from / re-checked out of the list
    bool bad = false;
    for (int t0 = 0; t0 < n; t0 += 32) {
        const int ci = t0 + lane;
        const float cv = ci < n ? dist(ci) : inf;
        bad = bad || (cv != cv);
        const bool want = ci < n && (cv < thr_v || (cv == thr_v && ci < thr_i));
        if (ci < n && !want) rej = fminf(rej, cv);
        unsigned mask = __ballot_sync(0xffffffffu, want);
        while (mask) {
            const int src = __ffs(mask) - 1;
            mask &= mask - 1;
            const float bv = __shfl_sync(0xffffffffu, cv, src);
            const int bi = __shfl_sync(0xffffffffu, ci, src);
            if (!(bv < thr_v || (bv == thr_v && bi < thr_i))) { ev = fminf(ev, bv); continue; }
            ev = fminf(ev, thr_v);                                // the current k-th falls out (inf while the list is filling)
            const int pos = __popc(__ballot_sync(0xffffffffu, lane < k && (lv < bv || (lv == bv && li < bi))));
            const float pv = __shfl_up_sync(0xffffffffu, lv, 1);
            const int pi = __shfl_up_sync(0xffffffffu, li, 1);
            if (lane > pos) { lv = pv; li = pi; }
            else if (lane == pos) { lv = bv; li = bi; }
            thr_v = __shfl_sync(0xffffffffu, lv, k - 1);
            thr_i = __shfl_sync(0xffffffffu, li, k - 1);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) rej = fminf(rej, __shfl_xor_sync(0xffffffffu, rej, o));
    const float runner_up = fminf(rej, ev);
    const float nv = __shfl_down_sync(0xffffffffu, lv, 1);
    const bool tie = (lane + 1 < k) && !(lv < nv);            // equal neighbours: not provably distinct
    const bool unfilled = lane < k && li == 0x7fffffff;
    const bool edge = !(thr_v < runner_up) && n > k;           // the k-th ties with (or is inf like) the best outsider
    if (__any_sync(0xffffffffu, tie || unfilled || bad) || edge) return false;
    if (lane < k) { val_out[lane] = lv; idx_out[lane] = li; }
    return true;
}

// Fast pass of knn_point: CTA = one cloud (staged in shared memory) x a chunk of its queries, 8 warps, distances computed
// on the fly, no per-row buffers -> many warps per SM hide the serial shuffle chains of the list insertions.
// Rows it cannot decide (ties) are flagged with idx[r*k] = -1 for knn_point_kernel.
constexpr int kKnnFastWarps = 8;
__global__ void __launch_bounds__(kKnnFastWarps * 32)
knn_point_fast_kernel(int n, int m, int c, int k, int q_per_cta, const float* __restrict__ xyz1, const float* __restrict__ xyz2,
                      float* __restrict__ val, int* __restrict__ idx) {
    extern __shared__ float smem_f[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int bi = blockIdx.y;
    const float* pg = xyz1 + (size_t)bi * n * c;
    for (int t = threadIdx.x; t < n * c; t += kKnnFastWarps * 32) smem_f[t] = __ldg(pg + t);
    __syncthreads();
    const float* p = smem_f;
    const int q0 = blockIdx.x * q_per_cta;
    const int q1 = min(m, q0 + q_per_cta);
    for (int qi = q0 + warp; qi < q1; qi += kKnnFastWarps) {
        const long long r = (long long)bi * m + qi;
        const float* q = xyz2 + r * c;
        bool done;
        if (c == 3) {
            const float qx = __ldg(q), qy = __ldg(q + 1), qz = __ldg(q + 2);
            done = knn_fast_path(n, k, [&](int t) {
                const float dx = __fsub_rn(p[3 * t], qx), dy = __fsub_rn(p[3 * t + 1], qy), dz = __fsub_rn(p[3 * t + 2], qz);
                return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
            }, lane, val + r * k, idx + r * k);
        } else {
            done = knn_fast_path(n, k, [&](int t) {
                float sacc = 0.f;
                for (int l = 0; l < c; ++l) {
                    const float df = __fsub_rn(p[(size_t)t * c + l], __ldg(q + l));
                    sacc = __fadd_rn(sacc, __fmul_rn(df, df));
                }
                return sacc;
            }, lane, val + r * k, idx + r * k);
        }
        if (!done && lane == 0) idx[r * k] = -1;
    }
}

// knn_point (tf_grouping.py:49-74) fused: distances sum_c (x1-x2)^2 (sequential, un-contracted) built straight
// into the warp's shared-memory row, then the fast path above or the reference's selection rounds; only the first k
// are written.  CTA = one cloud (staged once in shared memory) x a chunk of its queries, one query per warp at a time.
__global__ void __launch_bounds__(kSelWarps * 32)
knn_point_kernel(int n, int m, int c, int k, int q_per_cta, int stage_cloud, int only_flagged, const float* __restrict__ xyz1,
                 const float* __restrict__ xyz2, float* __restrict__ val, int* __restrict__ idx) {
    extern __shared__ float smem_f[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* v = smem_f + (size_t)warp * n * 2;
    int* id = reinterpret_cast<int*>(v + n);
    float* cloud = smem_f + (size_t)kSelWarps * n * 2;           // (n, c) when staged
    const int bi = blockIdx.y;
    const float* p = xyz1 + (size_t)bi * n * c;
    if (stage_cloud) {
        for (int t = threadIdx.x; t < n * c; t += kSelWarps * 32) cloud[t] = __ldg(p + t);
        __syncthreads();
        p = cloud;
    }
    const int q0 = blockIdx.x * q_per_cta;
    const int q1 = min(m, q0 + q_per_cta);
    for (int qi = q0 + warp; qi < q1; qi += kSelWarps) {
        const long long r = (long long)bi * m + qi;
        if (only_flagged && idx[r * k] != -1) continue;          // decided by knn_point_fast_kernel (warp-uniform)
        const float* q = xyz2 + r * c;
        if (c == 3) {
            const float qx = __ldg(q), qy = __ldg(q + 1), qz = __ldg(q + 2);
            for (int t = lane; t < n; t += 32) {
                const float dx = __fsub_rn(p[3 * t], qx), dy = __fsub_rn(p[3 * t + 1], qy), dz = __fsub_rn(p[3 * t + 2], qz);
                v[t] = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                id[t] = t;
            }
        } else {
            for (int t = lane; t < n; t += 32) {
                float sacc = 0.f;
                for (int l = 0; l < c; ++l) {
                    float df = __fsub_rn(p[(size_t)t * c + l], __ldg(q + l));
                    sacc = __fadd_rn(sacc, __fmul_rn(df, df));
                }
                v[t] = sacc; id[t] = t;
            }
        }
        __syncwarp();
        selection_rounds(n, k, v, id, lane);
        for (int t = lane; t < k; t += 32) { val[r * k + t] = v[t]; idx[r * k + t] = id[t]; }
        __syncwarp();
    }
}

static inline int grid_for(long long total, int block) {
    long long g = (total + block - 1) / block;
    long long cap = (long long)kNumSMs * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace psa

using namespace psa;

extern "C" int psa_query_ball_point(int b, int n, int m, float radius, int nsample, const float* xyz1,
                                    const float* xyz2, int* idx, int* pts_cnt, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && m >= 0, "QueryBallPoint: negative dimension (b=%d n=%d m=%d)", b, n, m);
    PSA_REQUIRE(nsample >= 0, "QueryBallPoint: nsample=%d", nsample);
    if (b == 0 || m == 0) return PSA_OK;
    PSA_REQUIRE(idx != nullptr || nsample == 0, "QueryBallPoint: null idx");
    PSA_REQUIRE((xyz1 != nullptr || n == 0) && xyz2 != nullptr, "QueryBallPoint: null input");
    // the spatial grid pays off once a CTA answers enough queries to amortise the counting sort
    const bool want_grid = bq_grid_fits(n) && n >= 256 && m >= 32;
    size_t smem = bq_smem_bytes(n, want_grid);
    PSA_SUPPORTED(smem <= 200 * 1024, "query_ball_point: n=%d exceeds the shared-memory resident limit", n);
    bool none = false;
    float thr = ball_query_threshold(radius, &none);
    // enough CTAs for ~2 waves of the SMs, at least two warp-batches of queries per CTA
    int chunks = (2 * kNumSMs + b - 1) / b;
    int q_per_cta = (m + chunks - 1) / chunks;
    // a CTA answers a multiple of 64 queries (8 warps x 8 queries per lane-per-slab step)
    const int qstep = kBqWarps * kBqSlabQueries;
    q_per_cta = ((q_per_cta + qstep - 1) / qstep) * qstep;
    dim3 grid((m + q_per_cta - 1) / q_per_cta, b);
    if (n <= 8 * kBqThreads) {
        PSA_CUDA(cudaFuncSetAttribute(ball_query_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ball_query_kernel<8><<<grid, kBqThreads, smem, as_stream(stream)>>>(n, m, nsample, radius, thr, none ? 1 : 0, want_grid ? 1 : 0,
                                                                            q_per_cta, xyz1, xyz2, idx, pts_cnt);
    } else {
        PSA_CUDA(cudaFuncSetAttribute(ball_query_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ball_query_kernel<16><<<grid, kBqThreads, smem, as_stream(stream)>>>(n, m, nsample, radius, thr, none ? 1 : 0, want_grid ? 1 : 0,
                                                                             q_per_cta, xyz1, xyz2, idx, pts_cnt);
    }
    return check_launch("ball_query_kernel");
}

extern "C" int psa_group_point(int b, int n, int c, int m, int nsample, const float* points, const int* idx,
                               float* out, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && c >= 0 && m >= 0 && nsample >= 0, "GroupPoint: negative dimension");
    long long rows_per_b = (long long)m * nsample;
    long long total = (long long)b * rows_per_b * c;
    if (total == 0) return PSA_OK;
    PSA_REQUIRE(points && idx && out, "GroupPoint: null buffer");
    cudaStream_t st = as_stream(stream);
    bool vec = (c % 4 == 0) && ((uintptr_t)points % 16 == 0) && ((uintptr_t)out % 16 == 0);
    if (vec) {
        long long tv = total / 4;
        group_point_kernel<float4><<<grid_for(tv, 256), 256, 0, st>>>(n, c / 4, rows_per_b, tv,
                                                                      reinterpret_cast<const float4*>(points), idx,
                                                                      reinterpret_cast<float4*>(out));
    } else {
        group_point_kernel<float><<<grid_for(total, 256), 256, 0, st>>>(n, c, rows_per_b, total, points, idx, out);
    }
    return check_launch("group_point_kernel");
}

extern "C" int psa_selection_sort(int b, int n, int m, int k, const float* dist, int* outi, float* out,
                                  psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && m >= 0 && k >= 0, "SelectionSort: negative dimension");
    long long rows = (long long)b * m;
    if (rows == 0 || n == 0) return PSA_OK;
    PSA_REQUIRE(dist && outi && out, "SelectionSort: null buffer");
    size_t smem = (size_t)kSelWarps * n * 2 * sizeof(float);
    PSA_SUPPORTED(smem <= 200 * 1024, "selection_sort: n=%d exceeds the shared-memory resident limit", n);
    PSA_CUDA(cudaFuncSetAttribute(selection_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = (int)((rows + kSelWarps - 1) / kSelWarps);
    if (grid > kNumSMs * 8) grid = kNumSMs * 8;
    selection_sort_kernel<<<grid, kSelWarps * 32, smem, as_stream(stream)>>>(rows, n, k, dist, outi, out);
    return check_launch("selection_sort_kernel");
}

extern "C" int psa_knn_point(int b, int n, int m, int c, int k, const float* xyz1, const float* xyz2, float* val,
                             int* idx, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && m >= 0 && c >= 0 && k >= 0, "knn_point: negative dimension");
    PSA_REQUIRE(k <= n, "knn_point: k=%d exceeds the number of dataset points n=%d", k, n);
    long long rows = (long long)b * m;
    if (rows == 0 || k == 0) return PSA_OK;
    PSA_REQUIRE(xyz1 && xyz2 && val && idx, "knn_point: null buffer");
    size_t smem = (size_t)kSelWarps * n * 2 * sizeof(float);
    PSA_SUPPORTED(smem <= 200 * 1024, "knn_point: n=%d exceeds the shared-memory resident limit", n);
    PSA_SUPPORTED(b <= 65535, "knn_point: b=%d exceeds gridDim.y", b);
    const size_t cloud_bytes = (size_t)n * c * sizeof(float);
    const int stage_cloud = (smem + cloud_bytes <= 100 * 1024) ? 1 : 0;      // keep two CTAs per SM
    if (stage_cloud) smem += cloud_bytes;
    PSA_CUDA(cudaFuncSetAttribute(knn_point_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int chunks = (2 * kNumSMs + b - 1) / b;
    int q_per_cta = (m + chunks - 1) / chunks;
    q_per_cta = ((q_per_cta + kKnnFastWarps - 1) / kKnnFastWarps) * kKnnFastWarps;
    dim3 grid((m + q_per_cta - 1) / q_per_cta, b);
    // fast pass first (distinct distances: the common case), then the reference's selection rounds for the rows it flagged
    const int fast = (k <= 32 && cloud_bytes <= 48 * 1024) ? 1 : 0;
    if (fast) {
        knn_point_fast_kernel<<<grid, kKnnFastWarps * 32, cloud_bytes, as_stream(stream)>>>(n, m, c, k, q_per_cta, xyz1, xyz2, val, idx);
        int rc = check_launch("knn_point_fast_kernel");
        if (rc != PSA_OK) return rc;
    }
    knn_point_kernel<<<grid, kSelWarps * 32, smem, as_stream(stream)>>>(n, m, c, k, q_per_cta, stage_cloud, fast, xyz1, xyz2, val, idx);
    return check_launch("knn_point_kernel");
}
