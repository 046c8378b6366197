// edgeconv_train.cu -- training mode of the single-layer EdgeConv (dgcnn/models/dgcnn.py:41-47, dgcnn/utils/tf_util.py:115-173,
// 462-499): out_ic = max_j relu(BN(y_ij)),  y_ij = [x_i, x_j - x_i] . W + b,  BN with batch statistics over all b*n*k edges.
//
//   W . [x_i ; x_j - x_i] = (W_a - W_b) . x_i + W_b . x_j,   so with  Q = x (W_a - W_b) + b  and  P = x W_b   (both (b*n, C_out))
//   y_ij = Q_i + P_nn(i,j)
//
// is one dense product over the b*n POINTS plus gather passes that recompute y_ij from L2 instead of a (b,n,k,2c) edge tensor and
// a (b,n,k,C_out) activation tensor.  y_ij is always evaluated as the single fp32 add Q_i + P_nn, so the statistics, the pooling, the
// tie detection of the max gradient and the backward all see the same bits.
//
// Gradient of the max: split evenly among the edges whose activated value equals the max bit for bit (torch.amax / TF reduce_max);
// ties are real -- the kNN graph contains the point itself and duplicated points.  Backward:
//   dz_ij = dout_ic / cnt_ic on the tied edges with a positive maximum, 0 elsewhere
//   dy_ij = ca dz_ij + cb y_ij + cc                     (psa_bn_bwd_coeffs' constants with rows = b*n*k)
//   dQ_i  = sum_j dy_ij               in j order
//   dP_p  = sum_{nn(i,j) = p} dy_ij   in ascending (i, j) order (stable counting sort of the graph, scatter.cu)
//   dW_a = x^T dQ,  dW_b = x^T (dP - dQ),  dx = dQ W_a^T + (dP - dQ) W_b^T
// Every reduction is partitioned by data (point tiles, reverse lists), never by which CTA ran what, and added in a fixed order: results
// are bit-reproducible.  One warp per centre point, lane = C_out / 32 consecutive channels.
#include <limits.h>

#include "mlp_internal.cuh"

namespace psa {
namespace {

constexpr int kEdgeWarps = 8;            // warps per block
constexpr int kEdgeTile = 64;            // centre points per statistics tile: the partial sums are indexed by tile
constexpr int kEdgeMaxN = 256;           // C_out limit (8 channels per lane)
constexpr int kEdgeMaxCloud = 51200;     // points per cloud of the counting sort (launch_group_csr)

// f(nb) for the k neighbours of one centre in j order; 32 indices per coalesced load, broadcast by shuffle
template <class F>
__device__ __forceinline__ void for_each_neighbour(const int* __restrict__ nn, int k, int lane, F&& f) {
    for (int j0 = 0; j0 < k; j0 += 32) {
        const int cnt = min(32, k - j0);
        const int mine = lane < cnt ? __ldg(nn + j0 + lane) : 0;
        for (int jj = 0; jj < cnt; ++jj) f(__shfl_sync(0xffffffffu, mine, jj));
    }
}

template <int VEC>
__device__ __forceinline__ void load_vec(float (&r)[VEC], const float* __restrict__ p) {
#pragma unroll
    for (int v = 0; v < VEC; ++v) r[v] = __ldg(p + v);
}

__device__ __forceinline__ float edge_act(float y, float s, float t) { return fmaxf(fmaf(y, s, t), 0.f); }   // train_pool_fwd_kernel's formula

__device__ __forceinline__ int load_tie(const void* ties, size_t o, bool wide) {
    return wide ? __ldg(reinterpret_cast<const int*>(ties) + o) : (int)__ldg(reinterpret_cast<const unsigned char*>(ties) + o);
}

// per-tile column partials (tile, 2, N) from the per-lane sums of the block's warps, added in warp order
template <int VEC>
__device__ __forceinline__ void store_tile_partial(float (*red)[2][kEdgeMaxN], const float (&a)[VEC], const float (&b)[VEC], int N,
                                                   float* __restrict__ dst) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int v = 0; v < VEC; ++v) { red[w][0][lane * VEC + v] = a[v]; red[w][1][lane * VEC + v] = b[v]; }
    __syncthreads();
    for (int e = threadIdx.x; e < 2 * N; e += kEdgeWarps * 32) {
        const int which = e / N, c = e - which * N;
        float t = 0.f;
#pragma unroll
        for (int ww = 0; ww < kEdgeWarps; ++ww) t += red[ww][which][c];
        dst[e] = t;
    }
    __syncthreads();
}

// forward statistics: partial[tile] = [sum y | sum y^2] over the edges of the tile's centre points
template <int VEC>
__global__ void __launch_bounds__(kEdgeWarps * 32)
edge_train_stats_kernel(long long points, int n, int k, int N, const float* __restrict__ PQ, const int* __restrict__ nn_idx, long long tiles,
                        float* __restrict__ partial) {
    __shared__ float red[kEdgeWarps][2][kEdgeMaxN];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, c0 = lane * VEC;
    for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        float s[VEC], q[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) { s[v] = 0.f; q[v] = 0.f; }
        for (int u = w; u < kEdgeTile; u += kEdgeWarps) {
            const long long p = tile * kEdgeTile + u;
            if (p >= points) break;
            const long long base = (p / n) * n;
            float a[VEC];
            load_vec<VEC>(a, PQ + (size_t)p * 2 * N + c0);
            for_each_neighbour(nn_idx + (size_t)p * k, k, lane, [&](int nb) {
                float bv[VEC];
                load_vec<VEC>(bv, PQ + (size_t)(base + nb) * 2 * N + N + c0);
#pragma unroll
                for (int v = 0; v < VEC; ++v) {
                    const float y = __fadd_rn(a[v], bv[v]);
                    s[v] += y;
                    q[v] = fmaf(y, y, q[v]);
                }
            });
        }
        store_tile_partial<VEC>(red, s, q, N, partial + (size_t)tile * 2 * N);
    }
}

// pooled_ic = max_j relu(BN(y_ij)),  ties_ic = #{j : relu(BN(y_ij)) == pooled_ic}
template <int VEC>
__global__ void __launch_bounds__(kEdgeWarps * 32)
edge_train_pool_kernel(long long points, int n, int k, int N, const float* __restrict__ PQ, const int* __restrict__ nn_idx,
                       const float* __restrict__ scale, const float* __restrict__ shift, float* __restrict__ pooled, void* __restrict__ ties) {
    const int lane = threadIdx.x & 31, c0 = lane * VEC;
    const bool wide = k > 255;
    float sc[VEC], sh[VEC];
    load_vec<VEC>(sc, scale + c0);
    load_vec<VEC>(sh, shift + c0);
    for (long long p = (long long)blockIdx.x * kEdgeWarps + (threadIdx.x >> 5); p < points; p += (long long)gridDim.x * kEdgeWarps) {
        const long long base = (p / n) * n;
        float a[VEC], mx[VEC];
        int cnt[VEC];
        load_vec<VEC>(a, PQ + (size_t)p * 2 * N + c0);
#pragma unroll
        for (int v = 0; v < VEC; ++v) { mx[v] = -1.f; cnt[v] = 0; }          // relu output >= 0: the first edge beats the sentinel
        for_each_neighbour(nn_idx + (size_t)p * k, k, lane, [&](int nb) {
            float bv[VEC];
            load_vec<VEC>(bv, PQ + (size_t)(base + nb) * 2 * N + N + c0);
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
                const float z = edge_act(__fadd_rn(a[v], bv[v]), sc[v], sh[v]);
                if (z > mx[v]) { mx[v] = z; cnt[v] = 1; }
                else if (z == mx[v]) ++cnt[v];
            }
        });
        const size_t o = (size_t)p * N + c0;
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
            pooled[o + v] = mx[v];
            if (wide) reinterpret_cast<int*>(ties)[o + v] = cnt[v];
            else reinterpret_cast<unsigned char*>(ties)[o + v] = (unsigned char)cnt[v];
        }
    }
}

// R_ic = dout_ic / ties_ic where pooled_ic > 0, else 0 (the max's gradient per tied edge), for the warp's VEC channels of point p
template <int VEC>
__device__ __forceinline__ void edge_route(size_t o, const float* __restrict__ pooled, const void* __restrict__ ties, bool wide,
                                           const float* __restrict__ dout, float* __restrict__ R, float (&mx)[VEC], float (&r)[VEC]) {
    load_vec<VEC>(mx, pooled + o);
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
        r[v] = mx[v] > 0.f ? __fdiv_rn(__ldg(dout + o + v), (float)load_tie(ties, o + v, wide)) : 0.f;
        R[o + v] = r[v];
    }
}

// frozen batch norm's backward pass 1: R alone (there are no batch-norm sums)
template <int VEC>
__global__ void __launch_bounds__(kEdgeWarps * 32)
edge_route_kernel(long long points, int k, int N, const float* __restrict__ pooled, const void* __restrict__ ties, const float* __restrict__ dout,
                  float* __restrict__ R) {
    const int c0 = (threadIdx.x & 31) * VEC;
    for (long long p = (long long)blockIdx.x * kEdgeWarps + (threadIdx.x >> 5); p < points; p += (long long)gridDim.x * kEdgeWarps) {
        float mx[VEC], r[VEC];
        edge_route<VEC>((size_t)p * N + c0, pooled, ties, k > 255, dout, R, mx, r);
    }
}

// backward pass 1: R (edge_route); partial[tile] = [sum dz | sum dz * xhat] over the tile's edges
template <int VEC>
__global__ void __launch_bounds__(kEdgeWarps * 32)
edge_train_bn_sums_kernel(long long points, int n, int k, int N, const float* __restrict__ PQ, const int* __restrict__ nn_idx,
                          const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ mean_inv,
                          const float* __restrict__ pooled, const void* __restrict__ ties, const float* __restrict__ dout, long long tiles,
                          float* __restrict__ R, float* __restrict__ partial) {
    __shared__ float red[kEdgeWarps][2][kEdgeMaxN];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, c0 = lane * VEC;
    const bool wide = k > 255;
    float sc[VEC], sh[VEC], mu[VEC], inv[VEC];
    load_vec<VEC>(sc, scale + c0);
    load_vec<VEC>(sh, shift + c0);
    load_vec<VEC>(mu, mean_inv + c0);
    load_vec<VEC>(inv, mean_inv + N + c0);
    for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        float sb[VEC], sg[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) { sb[v] = 0.f; sg[v] = 0.f; }
        for (int u = w; u < kEdgeTile; u += kEdgeWarps) {
            const long long p = tile * kEdgeTile + u;
            if (p >= points) break;
            const long long base = (p / n) * n;
            float a[VEC], mx[VEC], r[VEC];
            load_vec<VEC>(a, PQ + (size_t)p * 2 * N + c0);
            edge_route<VEC>((size_t)p * N + c0, pooled, ties, wide, dout, R, mx, r);
            for_each_neighbour(nn_idx + (size_t)p * k, k, lane, [&](int nb) {
                float bv[VEC];
                load_vec<VEC>(bv, PQ + (size_t)(base + nb) * 2 * N + N + c0);
#pragma unroll
                for (int v = 0; v < VEC; ++v) {
                    const float y = __fadd_rn(a[v], bv[v]);
                    if (edge_act(y, sc[v], sh[v]) == mx[v] && mx[v] > 0.f) {
                        sb[v] += r[v];
                        sg[v] = fmaf(r[v], (y - mu[v]) * inv[v], sg[v]);
                    }
                }
            });
        }
        store_tile_partial<VEC>(red, sb, sg, N, partial + (size_t)tile * 2 * N);
    }
}

// dz of edge (i, j): read from DZ (b*n*k, N) when given (a layer under another layer), else the max's gradient routed to the edges
// whose activation equals the pooled maximum (R = 0 where the maximum is not positive)
template <int VEC>
__device__ __forceinline__ float edge_dz(const float* __restrict__ DZ, size_t edge, int N, int c0, int v, float y, const float (&sc)[VEC],
                                         const float (&sh)[VEC], const float (&mx)[VEC], const float (&r)[VEC]) {
    return DZ != nullptr ? __ldg(DZ + edge * N + c0 + v) : (edge_act(y, sc[v], sh[v]) == mx[v] ? r[v] : 0.f);
}

// backward pass 2: G[p][0:N] = dQ_p = sum_j dy_pj in j order
template <int VEC>
__global__ void __launch_bounds__(kEdgeWarps * 32)
edge_train_dq_kernel(long long points, int n, int k, int N, const float* __restrict__ PQ, const int* __restrict__ nn_idx,
                     const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ coef,
                     const float* __restrict__ pooled, const float* __restrict__ R, const float* __restrict__ DZ, float* __restrict__ G) {
    const int lane = threadIdx.x & 31, c0 = lane * VEC;
    float sc[VEC], sh[VEC], ca[VEC], cb[VEC], cc[VEC];
    load_vec<VEC>(sc, scale + c0);
    load_vec<VEC>(sh, shift + c0);
    load_vec<VEC>(ca, coef + c0);
    load_vec<VEC>(cb, coef + N + c0);
    load_vec<VEC>(cc, coef + 2 * N + c0);
    for (long long p = (long long)blockIdx.x * kEdgeWarps + (threadIdx.x >> 5); p < points; p += (long long)gridDim.x * kEdgeWarps) {
        const long long base = (p / n) * n;
        const size_t o = (size_t)p * N + c0;
        float a[VEC], mx[VEC], r[VEC], acc[VEC];
        load_vec<VEC>(a, PQ + (size_t)p * 2 * N + c0);
        if (DZ == nullptr) {
            load_vec<VEC>(mx, pooled + o);
            load_vec<VEC>(r, R + o);
        }
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[v] = 0.f;
        size_t edge = (size_t)p * k;
        for_each_neighbour(nn_idx + (size_t)p * k, k, lane, [&](int nb) {
            float bv[VEC];
            load_vec<VEC>(bv, PQ + (size_t)(base + nb) * 2 * N + N + c0);
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
                const float y = __fadd_rn(a[v], bv[v]);
                const float dz = edge_dz<VEC>(DZ, edge, N, c0, v, y, sc, sh, mx, r);
                acc[v] += fmaf(ca[v], dz, fmaf(cb[v], y, cc[v]));
            }
            ++edge;
        });
#pragma unroll
        for (int v = 0; v < VEC; ++v) G[(size_t)p * 2 * N + c0 + v] = acc[v];
    }
}

// backward pass 3: G[p][N:2N] = dP_p - dQ_p,  dP_p = sum of dy_ij over the edges (i, j) with nn(i,j) = p, ascending (i, j)
template <int VEC>
__global__ void __launch_bounds__(kEdgeWarps * 32)
edge_train_dp_kernel(long long points, int n, int k, int N, const float* __restrict__ PQ, const float* __restrict__ scale,
                     const float* __restrict__ shift, const float* __restrict__ coef, const float* __restrict__ pooled,
                     const float* __restrict__ R, const float* __restrict__ DZ, const int* __restrict__ offsets, const int* __restrict__ list,
                     float* __restrict__ G) {
    const int lane = threadIdx.x & 31, c0 = lane * VEC;
    float sc[VEC], sh[VEC], ca[VEC], cb[VEC], cc[VEC];
    load_vec<VEC>(sc, scale + c0);
    load_vec<VEC>(sh, shift + c0);
    load_vec<VEC>(ca, coef + c0);
    load_vec<VEC>(cb, coef + N + c0);
    load_vec<VEC>(cc, coef + 2 * N + c0);
    const long long nk = (long long)n * k;
    for (long long p = (long long)blockIdx.x * kEdgeWarps + (threadIdx.x >> 5); p < points; p += (long long)gridDim.x * kEdgeWarps) {
        const long long cloud = p / n;
        const int jp = (int)(p - cloud * n);
        const int* off = offsets + (size_t)cloud * (n + 1);
        const int* lst = list + (size_t)cloud * nk;
        const int t0 = __ldg(off + jp), t1 = __ldg(off + jp + 1);
        float bp[VEC], acc[VEC];
        load_vec<VEC>(bp, PQ + (size_t)p * 2 * N + N + c0);
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[v] = 0.f;
        for (int e0 = t0; e0 < t1; e0 += 32) {
            const int cnt = min(32, t1 - e0);
            const int mine = lane < cnt ? __ldg(lst + e0 + lane) : 0;
            for (int jj = 0; jj < cnt; ++jj) {
                const int entry = __shfl_sync(0xffffffffu, mine, jj);                         // entry = i_local * k + j
                const long long i = cloud * n + entry / k;
                const size_t o = (size_t)i * N + c0, edge = (size_t)(cloud * nk + entry);
                float a[VEC], mx[VEC], r[VEC];
                load_vec<VEC>(a, PQ + (size_t)i * 2 * N + c0);
                if (DZ == nullptr) {
                    load_vec<VEC>(mx, pooled + o);
                    load_vec<VEC>(r, R + o);
                }
#pragma unroll
                for (int v = 0; v < VEC; ++v) {
                    const float y = __fadd_rn(a[v], bp[v]);
                    const float dz = edge_dz<VEC>(DZ, edge, N, c0, v, y, sc, sh, mx, r);
                    acc[v] += fmaf(ca[v], dz, fmaf(cb[v], y, cc[v]));
                }
            }
        }
        float* g = G + (size_t)p * 2 * N + c0;
#pragma unroll
        for (int v = 0; v < VEC; ++v) g[N + v] = acc[v] - g[v];
    }
}

size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
long long edge_tiles(long long rows) { return (rows + kEdgeTile - 1) / kEdgeTile; }
int edge_grid(long long rows) { return (int)((rows + kEdgeWarps - 1) / kEdgeWarps < 8LL * kNumSMs ? (rows + kEdgeWarps - 1) / kEdgeWarps : 8LL * kNumSMs); }
int tile_grid(long long tiles) { return (int)(tiles < 8LL * kNumSMs ? tiles : 8LL * kNumSMs); }

// workspace layouts (every segment 256-byte aligned)
struct FwdLayout {
    size_t wc, bias, part, dense, total;
    FwdLayout(int b, int n, int c, int N) {
        const long long rows = (long long)b * n;
        wc = 0;
        bias = wc + al256((size_t)c * 2 * N * sizeof(float));
        part = bias + al256((size_t)2 * N * sizeof(float));
        dense = part + al256((size_t)edge_tiles(rows) * 2 * N * sizeof(float));
        total = dense + al256(psa_train_dense_workspace_bytes(rows, c, 2 * N));
    }
};
// the tail shared with the two-layer backward (edge_layer_tail): G, the [W_a | W_b] copy, the reverse neighbour lists, the dense products
struct TailLayout {
    size_t g, w2, csr, dense, total;
    TailLayout(int b, int n, int c, int k, int N) {
        const long long rows = (long long)b * n;
        g = 0;
        w2 = g + al256((size_t)rows * 2 * N * sizeof(float));
        csr = w2 + al256((size_t)c * 2 * N * sizeof(float));
        dense = csr + al256(((size_t)b * (n + 1) + (size_t)rows * k) * sizeof(int));
        const size_t dw = psa_train_dense_workspace_bytes(rows, c, N), dx = psa_train_dense_workspace_bytes(rows, c, 2 * N);
        total = dense + al256(dw > dx ? dw : dx);
    }
};
struct BwdLayout {
    size_t r, coef, part, tail, total;
    BwdLayout(int b, int n, int c, int k, int N) {
        const long long rows = (long long)b * n;
        r = 0;
        coef = r + al256((size_t)rows * N * sizeof(float));
        part = coef + al256((size_t)3 * N * sizeof(float));
        tail = part + al256((size_t)edge_tiles(rows) * 2 * N * sizeof(float));
        total = tail + TailLayout(b, n, c, k, N).total;
    }
};

int check_dims(const char* who, int b, int n, int c, int k, int N) {
    PSA_REQUIRE(b >= 1 && n >= 1 && c >= 1 && k >= 1 && N >= 1, "%s: bad dims b=%d n=%d c=%d k=%d C_out=%d", who, b, n, c, k, N);
    PSA_SUPPORTED(N % 32 == 0 && N <= kEdgeMaxN, "%s: C_out=%d must be a multiple of 32, at most %d", who, N, kEdgeMaxN);
    PSA_SUPPORTED((long long)n * k <= INT_MAX, "%s: n*k = %lld edges per cloud exceed int32", who, (long long)n * k);
    return PSA_OK;
}

int check_ws(const char* who, const void* ws, size_t ws_bytes, size_t need) {
    PSA_REQUIRE(ws != nullptr && ws_bytes >= need, "%s: workspace of %zu bytes required (got %zu)", who, need, ws_bytes);
    PSA_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "%s: workspace must be 256-byte aligned", who);
    return PSA_OK;
}

psa_grad_in plain_grad(const float* dh, long long ld, int C) {
    psa_grad_in g = {};
    g.dh = dh; g.ld_dh = ld; g.pool_k = 1; g.C = C; g.mode = 0;
    return g;
}

}  // namespace
}  // namespace psa

using namespace psa;

#define PSA_EDGE_DISPATCH(KERNEL, GRID, SMEM, ...)                                                   \
    switch (N / 32) {                                                                              \
        case 1: KERNEL<1><<<GRID, kEdgeWarps * 32, SMEM, st>>>(__VA_ARGS__); break;                \
        case 2: KERNEL<2><<<GRID, kEdgeWarps * 32, SMEM, st>>>(__VA_ARGS__); break;                \
        case 3: KERNEL<3><<<GRID, kEdgeWarps * 32, SMEM, st>>>(__VA_ARGS__); break;                \
        case 4: KERNEL<4><<<GRID, kEdgeWarps * 32, SMEM, st>>>(__VA_ARGS__); break;                \
        case 5: KERNEL<5><<<GRID, kEdgeWarps * 32, SMEM, st>>>(__VA_ARGS__); break;                \
        case 6: KERNEL<6><<<GRID, kEdgeWarps * 32, SMEM, st>>>(__VA_ARGS__); break;                \
        case 7: KERNEL<7><<<GRID, kEdgeWarps * 32, SMEM, st>>>(__VA_ARGS__); break;                \
        default: KERNEL<8><<<GRID, kEdgeWarps * 32, SMEM, st>>>(__VA_ARGS__); break;               \
    }


size_t psa::edge_tail_workspace_bytes(int b, int n, int c, int k, int N) { return TailLayout(b, n, c, k, N).total; }

// dQ per centre, dP through the reverse neighbour lists, then dW = [x^T dQ ; x^T (dP - dQ)] and dx = [dQ | dP - dQ] . [W_a | W_b]^T
int psa::edge_layer_tail(int b, int n, int c, int k, int N, const float* x, const int* nn_idx, const float* W, const float* PQ, const float* scale,
                         const float* shift, const float* coef, const float* pooled, const float* R, const float* dz, float* dW, float* dx,
                         void* workspace, cudaStream_t st) {
    const long long rows = (long long)b * n;
    const TailLayout L(b, n, c, k, N);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    float* G = reinterpret_cast<float*>(ws + L.g);                  // (rows, 2N) = [dQ | dP - dQ]
    float* W2 = reinterpret_cast<float*>(ws + L.w2);                // (c, 2N) = [W_a | W_b]
    int* offsets = reinterpret_cast<int*>(ws + L.csr);
    int* list = offsets + (size_t)b * (n + 1);
    void* dense_ws = ws + L.dense;
    const size_t dense_bytes = L.total - L.dense;
    psa_stream_t stream = reinterpret_cast<psa_stream_t>(st);
    PSA_EDGE_DISPATCH(edge_train_dq_kernel, edge_grid(rows), 0, rows, n, k, N, PQ, nn_idx, scale, shift, coef, pooled, R, dz, G);
    int rc = check_launch("edge_train_dq_kernel");
    if (rc != PSA_OK) return rc;
    rc = launch_group_csr(b, n, n * k, nn_idx, offsets, list, st);
    if (rc != PSA_OK) return rc;
    PSA_EDGE_DISPATCH(edge_train_dp_kernel, edge_grid(rows), 0, rows, n, k, N, PQ, scale, shift, coef, pooled, R, dz, offsets, list, G);
    rc = check_launch("edge_train_dp_kernel");
    if (rc != PSA_OK) return rc;
    if (dW != nullptr) {
        // dW_a = x^T dQ, dW_b = x^T (dP - dQ): straight into the two row blocks of dW (2c, N)
        psa_act_in in = {};
        in.x = x; in.ld = c;
        const psa_grad_in gq = plain_grad(G, 2 * N, N), gd = plain_grad(G + N, 2 * N, N);
        rc = psa_train_dense_bwd_weight(rows, c, N, &in, &gq, dW, dense_ws, dense_bytes, stream);
        if (rc != PSA_OK) return rc;
        rc = psa_train_dense_bwd_weight(rows, c, N, &in, &gd, dW + (size_t)c * N, dense_ws, dense_bytes, stream);
        if (rc != PSA_OK) return rc;
    }
    // dx = [dQ | dP - dQ] . [W_a | W_b]^T: one product over 2N columns
    PSA_CUDA(cudaMemcpy2DAsync(W2, (size_t)2 * N * sizeof(float), W, (size_t)N * sizeof(float), (size_t)N * sizeof(float), c,
                               cudaMemcpyDeviceToDevice, st));
    PSA_CUDA(cudaMemcpy2DAsync(W2 + N, (size_t)2 * N * sizeof(float), W + (size_t)c * N, (size_t)N * sizeof(float), (size_t)N * sizeof(float), c,
                               cudaMemcpyDeviceToDevice, st));
    const psa_grad_in gg = plain_grad(G, 2 * N, 2 * N);
    return psa_train_dense_bwd_input(rows, c, 2 * N, &gg, W2, dx, c, 0, dense_ws, dense_bytes, stream);
}

int psa::frozen_coef(int N, const float* scale, float* coef, cudaStream_t st) {
    PSA_CUDA(cudaMemcpyAsync(coef, scale, (size_t)N * sizeof(float), cudaMemcpyDeviceToDevice, st));
    PSA_CUDA(cudaMemsetAsync(coef + N, 0, (size_t)2 * N * sizeof(float), st));
    return PSA_OK;
}

extern "C" size_t psa_edgeconv_train_workspace_bytes(int b, int n, int c, int k, int C_out) {
    if (b < 1 || n < 1 || c < 1 || k < 1 || C_out < 1 || C_out % 32 != 0 || C_out > kEdgeMaxN) return 0;
    const size_t f = FwdLayout(b, n, c, C_out).total, g = BwdLayout(b, n, c, k, C_out).total;
    return f > g ? f : g;
}

extern "C" int psa_edgeconv_train_fwd(int b, int n, int c, int k, int C_out, const float* x, const int* nn_idx, const float* W, const float* bias,
                                      float* PQ, float* stats, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    const int N = C_out;
    int rc = check_dims("edgeconv_train_fwd", b, n, c, k, N);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(x && nn_idx && W && PQ, "edgeconv_train_fwd: null buffer");
    rc = check_ws("edgeconv_train_fwd", workspace, workspace_bytes, psa_edgeconv_train_workspace_bytes(b, n, c, k, N));
    if (rc != PSA_OK) return rc;
    cudaStream_t st = as_stream(stream);
    const long long rows = (long long)b * n, tiles = edge_tiles(rows);
    const FwdLayout L(b, n, c, N);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    float* Wc = reinterpret_cast<float*>(ws + L.wc);
    float* bias2 = reinterpret_cast<float*>(ws + L.bias);
    float* partial = reinterpret_cast<float*>(ws + L.part);
    // [Q | P] = x . [W_a - W_b | W_b] + [b | 0]
    edge_wc_kernel<<<(c * 2 * N + 255) / 256, 256, 0, st>>>(c, N, W, Wc);
    rc = check_launch("edge_wc_kernel");
    if (rc != PSA_OK) return rc;
    PSA_CUDA(cudaMemsetAsync(bias2, 0, (size_t)2 * N * sizeof(float), st));
    if (bias != nullptr) PSA_CUDA(cudaMemcpyAsync(bias2, bias, (size_t)N * sizeof(float), cudaMemcpyDeviceToDevice, st));
    psa_act_in in = {};
    in.x = x; in.ld = c;
    rc = psa_train_dense_fwd(rows, c, 2 * N, &in, Wc, bias2, PQ, nullptr, ws + L.dense, L.total - L.dense, stream);
    if (rc != PSA_OK || stats == nullptr) return rc;            // no stats: frozen batch norm, PQ only
    PSA_EDGE_DISPATCH(edge_train_stats_kernel, tile_grid(tiles), 0, rows, n, k, N, PQ, nn_idx, tiles, partial);
    rc = check_launch("edge_train_stats_kernel");
    if (rc != PSA_OK) return rc;
    return reduce_partials((int)tiles, 2 * N, partial, stats, st);
}

extern "C" int psa_edgeconv_train_pool(int b, int n, int k, int C_out, const int* nn_idx, const float* PQ, const float* scale, const float* shift,
                                       float* pooled, void* ties, psa_stream_t stream) {
    const int N = C_out;
    int rc = check_dims("edgeconv_train_pool", b, n, 1, k, N);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(nn_idx && PQ && scale && shift && pooled && ties, "edgeconv_train_pool: null buffer");
    cudaStream_t st = as_stream(stream);
    const long long rows = (long long)b * n;
    PSA_EDGE_DISPATCH(edge_train_pool_kernel, edge_grid(rows), 0, rows, n, k, N, PQ, nn_idx, scale, shift, pooled, ties);
    return check_launch("edge_train_pool_kernel");
}

extern "C" int psa_edgeconv_train_bwd(int b, int n, int c, int k, int C_out, const float* x, const int* nn_idx, const float* W, const float* PQ,
                                      const float* scale, const float* shift, const float* gamma, const float* mean_inv, const float* pooled,
                                      const void* ties, const float* dout, float* dW, float* dgamma, float* dbeta, float* dx, void* workspace,
                                      size_t workspace_bytes, psa_stream_t stream) {
    const int N = C_out;
    int rc = check_dims("edgeconv_train_bwd", b, n, c, k, N);
    if (rc != PSA_OK) return rc;
    PSA_SUPPORTED(n <= kEdgeMaxCloud, "edgeconv_train_bwd: n=%d points per cloud exceed %d (reverse neighbour lists)", n, kEdgeMaxCloud);
    PSA_REQUIRE(x && nn_idx && W && PQ && scale && shift && gamma && mean_inv && pooled && ties && dout && dW && dgamma && dbeta && dx,
                "edgeconv_train_bwd: null buffer");
    rc = check_ws("edgeconv_train_bwd", workspace, workspace_bytes, psa_edgeconv_train_workspace_bytes(b, n, c, k, N));
    if (rc != PSA_OK) return rc;
    cudaStream_t st = as_stream(stream);
    const long long rows = (long long)b * n, tiles = edge_tiles(rows);
    const BwdLayout L(b, n, c, k, N);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    float* R = reinterpret_cast<float*>(ws + L.r);                  // (rows, N) routed gradient of a tied edge
    float* coef = reinterpret_cast<float*>(ws + L.coef);            // (3, N) = ca, cb, cc
    float* partial = reinterpret_cast<float*>(ws + L.part);
    // batch-norm sums over all b*n*k edges -> dgamma, dbeta, ca, cb, cc
    PSA_EDGE_DISPATCH(edge_train_bn_sums_kernel, tile_grid(tiles), 0, rows, n, k, N, PQ, nn_idx, scale, shift, mean_inv, pooled, ties, dout, tiles,
                      R, partial);
    rc = check_launch("edge_train_bn_sums_kernel");
    if (rc != PSA_OK) return rc;
    rc = launch_bn_bwd_final((int)tiles, N, rows * k, partial, gamma, mean_inv, dgamma, dbeta, coef, coef + N, coef + 2 * N, st);
    if (rc != PSA_OK) return rc;
    return edge_layer_tail(b, n, c, k, N, x, nn_idx, W, PQ, scale, shift, coef, pooled, R, nullptr, dW, dx, ws + L.tail, st);
}

extern "C" int psa_edgeconv_frozen_bwd(int b, int n, int c, int k, int C_out, const float* x, const int* nn_idx, const float* W, const float* PQ,
                                       const float* scale, const float* shift, const float* pooled, const void* ties, const float* dout, float* dx,
                                       void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    const int N = C_out;
    int rc = check_dims("edgeconv_frozen_bwd", b, n, c, k, N);
    if (rc != PSA_OK) return rc;
    PSA_SUPPORTED(n <= kEdgeMaxCloud, "edgeconv_frozen_bwd: n=%d points per cloud exceed %d (reverse neighbour lists)", n, kEdgeMaxCloud);
    PSA_REQUIRE(x && nn_idx && W && PQ && scale && shift && pooled && ties && dout && dx, "edgeconv_frozen_bwd: null buffer");
    rc = check_ws("edgeconv_frozen_bwd", workspace, workspace_bytes, psa_edgeconv_train_workspace_bytes(b, n, c, k, N));
    if (rc != PSA_OK) return rc;
    cudaStream_t st = as_stream(stream);
    const long long rows = (long long)b * n;
    const BwdLayout L(b, n, c, k, N);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    float* R = reinterpret_cast<float*>(ws + L.r);
    float* coef = reinterpret_cast<float*>(ws + L.coef);
    // the max's gradient routed to the tied edges (no batch-norm sums), then dy = scale * dz
    PSA_EDGE_DISPATCH(edge_route_kernel, edge_grid(rows), 0, rows, k, N, pooled, ties, dout, R);
    rc = check_launch("edge_route_kernel");
    if (rc != PSA_OK) return rc;
    rc = frozen_coef(N, scale, coef, st);
    if (rc != PSA_OK) return rc;
    return edge_layer_tail(b, n, c, k, N, x, nn_idx, W, PQ, scale, shift, coef, pooled, R, nullptr, nullptr, dx, ws + L.tail, st);
}
