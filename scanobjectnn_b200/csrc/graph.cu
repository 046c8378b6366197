// graph.cu -- DGCNN graph functions for sm_90a: pairwise_distance, knn (top-k), the fused kNN graph that never
// materialises the (B,N,N) matrix, and get_edge_feature.
//
// Reference: dgcnn/utils/tf_util.py:638-706 -- tf.matmul + reduce_sum + transpose (a (B,N,N) fp32 matrix, 512 MiB at
// B=32,N=2048, written and read back five times per forward), tf.nn.top_k, tf.gather/tile/concat.
// Arithmetic contract (the reference's cuBLAS/top_k order is unpinned, SURVEY 8c; canonical order shared with
// oracle/psa_oracle.c:orc_dgcnn_knn):  dot = fma chain over c ascending from 0;  sq = fma chain likewise;
// adj = (sq_i + (-2*dot)) + sq_j;  neighbours ascending by (adj, index), self included.
#include "common.cuh"

namespace psa {

constexpr int kPdTile = 64;      // 64x64 outputs per CTA, 256 threads, 4x4 per thread
constexpr int kPdCk = 32;        // channels staged per step

__global__ void __launch_bounds__(256)
pairwise_distance_kernel(int n, int c, const float* __restrict__ x, float* __restrict__ adj) {
    __shared__ float Xi[kPdTile][kPdCk + 1];
    __shared__ float Xj[kPdTile][kPdCk + 1];
    const int cloud = blockIdx.z;
    const int i0 = blockIdx.y * kPdTile, j0 = blockIdx.x * kPdTile;
    const float* xb = x + (size_t)cloud * n * c;
    // thread = 8 rows (ty + 8a) x 2 columns (tx + 32 b2): a warp's stores are 128 contiguous bytes of one adj row
    const int ty = threadIdx.x >> 5, tx = threadIdx.x & 31;
    float dot[8][2], sqi[8], sqj[2];
#pragma unroll
    for (int a = 0; a < 8; ++a) {
        sqi[a] = 0.f;
        dot[a][0] = dot[a][1] = 0.f;
    }
    sqj[0] = sqj[1] = 0.f;
    for (int c0 = 0; c0 < c; c0 += kPdCk) {
        const int cc = min(kPdCk, c - c0);
        __syncthreads();
        for (int s = threadIdx.x; s < kPdTile * kPdCk; s += 256) {
            int r = s / kPdCk, l = s - r * kPdCk;
            Xi[r][l] = (i0 + r < n && l < cc) ? __ldg(xb + (size_t)(i0 + r) * c + c0 + l) : 0.f;
            Xj[r][l] = (j0 + r < n && l < cc) ? __ldg(xb + (size_t)(j0 + r) * c + c0 + l) : 0.f;
        }
        __syncthreads();
        for (int l = 0; l < cc; ++l) {
            const float b0 = Xj[tx][l], b1 = Xj[tx + 32][l];
            sqj[0] = __fmaf_rn(b0, b0, sqj[0]);
            sqj[1] = __fmaf_rn(b1, b1, sqj[1]);
#pragma unroll
            for (int a = 0; a < 8; ++a) {
                const float ai = Xi[ty + 8 * a][l];             // warp-uniform address: broadcast
                sqi[a] = __fmaf_rn(ai, ai, sqi[a]);
                dot[a][0] = __fmaf_rn(ai, b0, dot[a][0]);
                dot[a][1] = __fmaf_rn(ai, b1, dot[a][1]);
            }
        }
    }
#pragma unroll
    for (int a = 0; a < 8; ++a) {
        const int i = i0 + ty + 8 * a;
        if (i >= n) continue;
#pragma unroll
        for (int b2 = 0; b2 < 2; ++b2) {
            const int j = j0 + tx + 32 * b2;
            if (j < n)     // streaming store: the (B,N,N) matrix is larger than L2 and read once
                __stcs(adj + ((size_t)cloud * n + i) * n + j, __fadd_rn(__fadd_rn(sqi[a], __fmul_rn(-2.0f, dot[a][b2])), sqj[b2]));
        }
    }
}

// k rounds of "smallest (value, index) strictly greater than the last pick" over a row resident in shared memory
__device__ __forceinline__ void topk_rounds(const float* row, int ncols, int k, int* __restrict__ out, int lane) {
    float lv = 0.f;
    int li = -1;
    for (int s = 0; s < k; ++s) {
        float bv = 0.f;
        int bi = -1;
        for (int t = lane; t < ncols; t += 32) {
            const float v = row[t];
            const bool after = (li < 0) || (v > lv) || (v == lv && t > li);
            if (after && (bi < 0 || v < bv)) { bv = v; bi = t; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi >= 0 && (bi < 0 || ov < bv || (ov == bv && oi < bi))) { bv = ov; bi = oi; }
        }
        if (lane == 0) out[s] = bi < 0 ? 0 : bi;
        lv = bv; li = bi;
    }
}

constexpr int kTopkWarps = 4;

// top-k of a row streamed ONCE from global memory (k <= 32): the warp keeps the k best as a sorted list, one (value, index)
// per lane; a candidate enters only if it beats the k-th by (value, index) -- candidates arrive in index order, so equal
// values keep the lower index first like tf.nn.top_k -- placed by popc(ballot(list < cand)) and a shuffle-up shift.
// Expected k(1 + ln(n/k)) insertions per row instead of k full passes.
constexpr int kTopk2Warps = 8;
__global__ void __launch_bounds__(kTopk2Warps * 32)
knn_topk_stream_kernel(long long rows, int ncols, int k, const float* __restrict__ adj, int* __restrict__ nn_idx) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float inf = __int_as_float(0x7f800000);
    for (long long r = (long long)blockIdx.x * kTopk2Warps + warp; r < rows; r += (long long)gridDim.x * kTopk2Warps) {
        const float* row = adj + r * ncols;
        float lv = inf;
        int li = 0x7fffffff;                               // empty slot: loses against every real (value, index)
        float thr_v = inf;
        int thr_i = 0x7fffffff;
        float nxt = lane < ncols ? __ldcs(row + lane) : 0.f;
        for (int t0 = 0; t0 < ncols; t0 += 32) {
            const float cv = nxt;
            const int ci = t0 + lane;
            if (t0 + 32 + lane < ncols) nxt = __ldcs(row + t0 + 32 + lane);
            unsigned mask = __ballot_sync(0xffffffffu, ci < ncols && (cv < thr_v || (cv == thr_v && ci < thr_i)));
            while (mask) {
                const int src = __ffs(mask) - 1;
                mask &= mask - 1;
                const float bv = __shfl_sync(0xffffffffu, cv, src);
                const int bi = __shfl_sync(0xffffffffu, ci, src);
                if (!(bv < thr_v || (bv == thr_v && bi < thr_i))) continue;          // the k-th best tightened meanwhile
                const int pos = __popc(__ballot_sync(0xffffffffu, lane < k && (lv < bv || (lv == bv && li < bi))));
                const float pv = __shfl_up_sync(0xffffffffu, lv, 1);
                const int pi = __shfl_up_sync(0xffffffffu, li, 1);
                if (lane > pos) { lv = pv; li = pi; }
                else if (lane == pos) { lv = bv; li = bi; }
                thr_v = __shfl_sync(0xffffffffu, lv, k - 1);
                thr_i = __shfl_sync(0xffffffffu, li, k - 1);
            }
        }
        if (lane < k) nn_idx[r * k + lane] = li == 0x7fffffff ? 0 : li;
    }
}

__global__ void __launch_bounds__(kTopkWarps * 32)
knn_topk_kernel(long long rows, int ncols, int k, const float* __restrict__ adj, int* __restrict__ nn_idx) {
    extern __shared__ float smem_f[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* row = smem_f + (size_t)warp * ncols;
    for (long long r = (long long)blockIdx.x * kTopkWarps + warp; r < rows; r += (long long)gridDim.x * kTopkWarps) {
        for (int t = lane; t < ncols; t += 32) row[t] = __ldg(adj + r * ncols + t);
        __syncwarp();
        topk_rounds(row, ncols, k, nn_idx + r * k, lane);
        __syncwarp();
    }
}

// Fused kNN graph: CTA = 64 queries of one cloud against all candidates, 64 at a time.
//   distances  4x4 register tiles (4 consecutive rows x 4 consecutive columns per thread) over TRANSPOSED shared-memory
//              channel chunks, so one LDS.128 feeds four rows / columns; dot and |x|^2 are fma chains over c ascending
//              (the canonical order of oracle/psa_oracle.c:orc_dgcnn_knn), adj = (sq_i + (-2 dot)) + sq_j -> a 64x64 tile
//              in shared memory: the (B,N,N) matrix never exists, HBM sees B*(4NC + 4Nk) bytes;
//   selection  each warp owns 8 query rows whose current k best stay sorted in REGISTERS (one list element per lane) for the
//              whole kernel.  The first tile is ranked by counting (no insertions); afterwards a candidate enters only if
//              it beats the k-th (strict '<': candidates arrive in index order, so equal values keep the lower index first,
//              like tf.nn.top_k), found by ballot, placed by popc(ballot(list <= cand)) and a shuffle-up shift.
constexpr int kKgQ = 64, kKgC = 64, kKgCk = 32, kKgLd = 68;

__global__ void __launch_bounds__(256)
knn_graph_kernel(int n, int c, int k, const float* __restrict__ x, int* __restrict__ nn_idx) {
    extern __shared__ __align__(16) float smem_f[];
    const int cq = (c + 3) & ~3;
    float* XqT = smem_f;                                 // [cq][68]  query features, transposed
    float* XjT = XqT + (size_t)cq * kKgLd;               // [32][68]  candidate chunk, transposed
    float* D = XjT + kKgCk * kKgLd;                      // [64][65]  adj tile
    float* Tv = D + kKgQ * (kKgC + 1);                   // [8 warps][64] scratch for the first-tile ranking
    int* Ti = reinterpret_cast<int*>(Tv + 8 * 64);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ty = tid >> 4, tx = tid & 15;
    const int cloud = blockIdx.y, q0 = blockIdx.x * kKgQ;
    const float* xb = x + (size_t)cloud * n * c;
    const float inf = __int_as_float(0x7f800000);
    for (int sidx = tid; sidx < kKgQ * c; sidx += 256) {
        const int r = sidx / c, l = sidx - r * c;
        XqT[l * kKgLd + r] = (q0 + r < n) ? __ldg(xb + (size_t)(q0 + r) * c + l) : 0.f;
    }
    __syncthreads();
    float sqi[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        float sq = 0.f;
        for (int l = 0; l < c; ++l) { const float v = XqT[l * kKgLd + ty * 4 + a]; sq = __fmaf_rn(v, v, sq); }
        sqi[a] = sq;
    }
    float lv[8];          // this lane's element of the sorted list of row warp*8+i
    int li[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { lv[i] = inf; li[i] = 0; }

    for (int j0 = 0; j0 < n; j0 += kKgC) {
        float dot[4][4], sqj[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            sqj[a] = 0.f;
#pragma unroll
            for (int b2 = 0; b2 < 4; ++b2) dot[a][b2] = 0.f;
        }
        for (int c0 = 0; c0 < c; c0 += kKgCk) {
            const int cc = min(kKgCk, c - c0);
            __syncthreads();
            for (int s0 = tid; s0 < kKgC * kKgCk; s0 += 256 * 4) {        // 4 independent loads in flight per thread
                float v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int sidx = s0 + u * 256, r = sidx / kKgCk, l = sidx - r * kKgCk;
                    v[u] = (sidx < kKgC * kKgCk && j0 + r < n && l < cc) ? __ldg(xb + (size_t)(j0 + r) * c + c0 + l) : 0.f;
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int sidx = s0 + u * 256, r = sidx / kKgCk, l = sidx - r * kKgCk;
                    if (sidx < kKgC * kKgCk) XjT[l * kKgLd + r] = v[u];
                }
            }
            __syncthreads();
            for (int l = 0; l < cc; ++l) {
                const float4 a4 = *reinterpret_cast<const float4*>(XqT + (c0 + l) * kKgLd + ty * 4);
                const float4 b4 = *reinterpret_cast<const float4*>(XjT + l * kKgLd + tx * 4);
                const float ai[4] = {a4.x, a4.y, a4.z, a4.w}, bj[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    sqj[a] = __fmaf_rn(bj[a], bj[a], sqj[a]);
#pragma unroll
                    for (int b2 = 0; b2 < 4; ++b2) dot[a][b2] = __fmaf_rn(ai[a], bj[b2], dot[a][b2]);
                }
            }
        }
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b2 = 0; b2 < 4; ++b2)
                D[(ty * 4 + a) * (kKgC + 1) + tx * 4 + b2] = __fadd_rn(__fadd_rn(sqi[a], __fmul_rn(-2.0f, dot[a][b2])), sqj[b2]);
        __syncthreads();
        // ---- selection: warp w owns query rows 8w..8w+7 ----
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = warp * 8 + i;
            if (q0 + r >= n) continue;                                     // warp-uniform
            const float cv0 = D[r * (kKgC + 1) + lane], cv1 = D[r * (kKgC + 1) + 32 + lane];
            const int ci0 = j0 + lane, ci1 = j0 + 32 + lane;
            if (j0 == 0) {
                // first tile: rank every candidate by counting (value, then index) and drop the k best into the list
                float* tv = Tv + warp * 64;
                int* ti = Ti + warp * 64;
                int r0 = 0, r1 = 0;
                const float v0 = ci0 < n ? cv0 : inf, v1 = ci1 < n ? cv1 : inf;
                for (int j = 0; j < 64; ++j) {
                    const float o = (j0 + j < n) ? D[r * (kKgC + 1) + j] : inf;      // broadcast
                    r0 += (o < v0 || (o == v0 && j < lane)) ? 1 : 0;
                    r1 += (o < v1 || (o == v1 && j < 32 + lane)) ? 1 : 0;
                }
                tv[r0] = v0; ti[r0] = ci0;
                tv[r1] = v1; ti[r1] = ci1;
                __syncwarp();
                lv[i] = lane < k ? tv[lane] : inf;
                li[i] = lane < k ? ti[lane] : 0;
                __syncwarp();
                continue;
            }
            float thr = __shfl_sync(0xffffffffu, lv[i], k - 1);
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const float cv = half ? cv1 : cv0;
                const int ci = half ? ci1 : ci0;
                unsigned mask = __ballot_sync(0xffffffffu, ci < n && cv < thr);
                while (mask) {
                    const int src = __ffs(mask) - 1;
                    mask &= mask - 1;
                    const float bv = __shfl_sync(0xffffffffu, cv, src);
                    const int bi = __shfl_sync(0xffffffffu, ci, src);
                    if (!(bv < thr)) continue;                             // the k-th best tightened meanwhile
                    const int pos = __popc(__ballot_sync(0xffffffffu, lane < k && lv[i] <= bv));
                    const float pv = __shfl_up_sync(0xffffffffu, lv[i], 1);
                    const int pi = __shfl_up_sync(0xffffffffu, li[i], 1);
                    if (lane > pos) { lv[i] = pv; li[i] = pi; }
                    else if (lane == pos) { lv[i] = bv; li[i] = bi; }
                    if (lane >= k) lv[i] = inf;
                    thr = __shfl_sync(0xffffffffu, lv[i], k - 1);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int r = warp * 8 + i;
        if (q0 + r < n && lane < k) nn_idx[((size_t)cloud * n + q0 + r) * k + lane] = li[i];
    }
}

// edge[b,i,j,:] = [x_i, x_{nn(i,j)} - x_i], vectorised: 2c/4 threads per edge row, one index computation per row,
// float4 streaming stores (the (B,N,k,2C) tensor is written once and is larger than L2)
__global__ void __launch_bounds__(256)
edge_feature_vec_kernel(int n, int c4, int k, long long rows, const float4* __restrict__ x, const int* __restrict__ nn_idx,
                        float4* __restrict__ out) {
    const int tpr = 2 * c4;                                   // threads per edge row
    const int rpb = 256 / tpr;                                // rows per block iteration
    const int lr = threadIdx.x / tpr, l = threadIdx.x - lr * tpr;
    if (lr >= rpb) return;
    for (long long row = (long long)blockIdx.x * rpb + lr; row < rows; row += (long long)gridDim.x * rpb) {
        const long long pi = row / k;                         // b*n + i
        const float4 xi = __ldg(x + pi * c4 + (l < c4 ? l : l - c4));
        float4 v = xi;
        if (l >= c4) {
            const long long bi = pi / n;
            const int j = __ldg(nn_idx + row);
            const float4 xj = __ldg(x + (bi * n + j) * c4 + (l - c4));
            v = make_float4(xj.x - xi.x, xj.y - xi.y, xj.z - xi.z, xj.w - xi.w);
        }
        __stcs(out + row * tpr + l, v);
    }
}

// edge[b,i,j,:] = [x_i, x_{nn(i,j)} - x_i]
__global__ void edge_feature_kernel(int n, int c, int k, long long total, const float* __restrict__ x,
                                    const int* __restrict__ nn_idx, float* __restrict__ out) {
    const int c2 = 2 * c;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        long long row = e / c2;           // (b*n + i)*k + j
        int l = (int)(e - row * c2);
        long long pi = row / k;           // b*n + i
        long long bi = pi / n;
        if (l < c) {
            out[e] = __ldg(x + pi * c + l);
        } else {
            int j = __ldg(nn_idx + row);
            out[e] = __ldg(x + (bi * n + j) * c + (l - c)) - __ldg(x + pi * c + (l - c));
        }
    }
}

static inline int grid_for(long long total, int block) {
    long long g = (total + block - 1) / block;
    long long cap = (long long)kNumSMs * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace psa

using namespace psa;

extern "C" int psa_pairwise_distance(int b, int n, int c, const float* x, float* adj, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && c >= 0, "pairwise_distance: negative dimension");
    if (b == 0 || n == 0) return PSA_OK;
    PSA_REQUIRE((x || c == 0) && adj, "pairwise_distance: null buffer");
    PSA_SUPPORTED(b <= 65535, "pairwise_distance: b=%d exceeds gridDim.z", b);
    dim3 grid((n + kPdTile - 1) / kPdTile, (n + kPdTile - 1) / kPdTile, b);
    pairwise_distance_kernel<<<grid, 256, 0, as_stream(stream)>>>(n, c, x, adj);
    return check_launch("pairwise_distance_kernel");
}

extern "C" int psa_knn_topk(int b, int n, int ncols, int k, const float* adj, int* nn_idx, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && ncols >= 0 && k >= 0, "knn: negative dimension");
    PSA_REQUIRE(k <= ncols, "knn: k=%d exceeds the row length %d (tf.nn.top_k: input must have at least k columns)", k, ncols);
    long long rows = (long long)b * n;
    if (rows == 0 || k == 0) return PSA_OK;
    PSA_REQUIRE(adj && nn_idx, "knn: null buffer");
    if (k <= 32) {
        long long g2 = (rows + kTopk2Warps - 1) / kTopk2Warps;
        if (g2 > (long long)kNumSMs * 16) g2 = (long long)kNumSMs * 16;
        knn_topk_stream_kernel<<<(int)g2, kTopk2Warps * 32, 0, as_stream(stream)>>>(rows, ncols, k, adj, nn_idx);
        return check_launch("knn_topk_stream_kernel");
    }
    size_t smem = (size_t)kTopkWarps * ncols * sizeof(float);
    PSA_SUPPORTED(smem <= 200 * 1024, "knn: row length %d exceeds the shared-memory resident limit", ncols);
    PSA_CUDA(cudaFuncSetAttribute(knn_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = (int)((rows + kTopkWarps - 1) / kTopkWarps);
    if (grid > kNumSMs * 16) grid = kNumSMs * 16;
    knn_topk_kernel<<<grid, kTopkWarps * 32, smem, as_stream(stream)>>>(rows, ncols, k, adj, nn_idx);
    return check_launch("knn_topk_kernel");
}

extern "C" int psa_knn_graph(int b, int n, int c, int k, const float* x, int* nn_idx, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && c >= 0 && k >= 0, "knn_graph: negative dimension");
    PSA_REQUIRE(k <= n || b == 0, "knn_graph: k=%d exceeds the number of points n=%d", k, n);
    if (b == 0 || n == 0 || k == 0) return PSA_OK;
    PSA_REQUIRE((x || c == 0) && nn_idx, "knn_graph: null buffer");
    PSA_SUPPORTED(b <= 65535, "knn_graph: b=%d exceeds gridDim.y", b);
    PSA_SUPPORTED(k <= 32, "knn_graph: k=%d exceeds the 32 entries a warp keeps per query", k);
    size_t smem = ((size_t)((c + 3) & ~3) * kKgLd + (size_t)kKgCk * kKgLd + (size_t)kKgQ * (kKgC + 1) + 2 * 8 * 64) * sizeof(float);
    PSA_SUPPORTED(smem <= 200 * 1024, "knn_graph: c=%d exceeds the shared-memory resident limit", c);
    PSA_CUDA(cudaFuncSetAttribute(knn_graph_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((n + kKgQ - 1) / kKgQ, b);
    knn_graph_kernel<<<grid, 256, smem, as_stream(stream)>>>(n, c, k, x, nn_idx);
    return check_launch("knn_graph_kernel");
}

extern "C" int psa_get_edge_feature(int b, int n, int c, int k, const float* x, const int* nn_idx, float* out,
                                    psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && c >= 0 && k >= 0, "get_edge_feature: negative dimension");
    long long total = (long long)b * n * k * 2 * c;
    if (total == 0) return PSA_OK;
    PSA_REQUIRE(x && nn_idx && out, "get_edge_feature: null buffer");
    if ((c % 4) == 0 && c <= 512 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {
        const long long rows = (long long)b * n * k;
        const int rpb = 256 / (c / 2);
        long long g = (rows + rpb - 1) / rpb;
        if (g > (long long)kNumSMs * 32) g = (long long)kNumSMs * 32;
        edge_feature_vec_kernel<<<(int)g, 256, 0, as_stream(stream)>>>(n, c / 4, k, rows, reinterpret_cast<const float4*>(x), nn_idx,
                                                                       reinterpret_cast<float4*>(out));
        return check_launch("edge_feature_vec_kernel");
    }
    edge_feature_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(n, c, k, total, x, nn_idx, out);
    return check_launch("edge_feature_kernel");
}
