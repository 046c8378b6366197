// mlp.cu -- grouped per-point shared MLP with the neighbourhood gather fused in front and the channel-wise
// max-pool fused behind it (fp32 FMA path, sm_90a).
//
// Reference: pointnet_sa_module (pointnet2/utils/pointnet_util.py:87-154) = group_point + tile/sub + concat,
// then three tf_util.conv2d 1x1 (+bias+BN+ReLU, pointnet2/utils/tf_util.py:120-185) and tf.reduce_max -- each a
// separate TF/cuDNN pass over the materialised (B,m,K,C) tensors (up to 256 MiB per layer at B=32,N=2048).
// DGCNN's EdgeConv (dgcnn/utils/tf_util.py:674-706 + dgcnn/models/dgcnn.py:31-80) has the same shape.
//
// Here one CTA owns a tile of up to 128 grouped rows (G = 128/K neighbourhoods), gathers them ONCE from HBM/L2
// into shared memory, runs the whole MLP chain on-chip (activations ping-pong between two row-major shared
// buffers, weights streamed through a cp.async double buffer and served from L2), and reduces the last layer's
// output over each neighbourhood in the epilogue.  HBM sees: idx + the gathered source rows + the pooled output.
//
// Arithmetic: fp32 FMA chains, k ascending in the shared-memory channel order (SA rows are stored
// [features..., dx,dy,dz] so the feature part stays 16-byte aligned; weight rows are permuted to match).
// Parity target vs the fp32/fp64 restatement: 1e-5 (see tests/test_mlp_gpu.py).
#include <float.h>

#include "common.cuh"
#include "mlp_internal.cuh"

namespace psa {

constexpr int kMlpThreads = 256;
constexpr int BM = 128;   // rows per tile
constexpr int BK = 16;    // k-rows per staged weight chunk
constexpr int BN_MAX = 128;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// order-preserving float <-> int map (involution) so shared/global atomicMax(int) implements float max
__device__ __forceinline__ int f2ord(float f) {
    int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

// Stage rows [k0, k0+BK) x cols [n0, n0+BN) of W (global, [K][N] row-major) into Ws[BK][BN]; zero beyond K / N.
// perm_c >= 0: shared-memory channel kk maps to weight row (kk < perm_c ? kk + 3 : kk - perm_c)  (SA layer 0).
template <int BN>
__device__ __forceinline__ void load_w_chunk(float* Ws, const float* __restrict__ W, int K, int N, int k0, int n0,
                                             int perm_c, int tid) {
    constexpr int SLOTS = BK * BN / 4;
    const bool row_aligned = ((N & 3) == 0) && ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
#pragma unroll
    for (int s = tid; s < SLOTS; s += kMlpThreads) {
        const int kk = s / (BN / 4);
        const int c4 = (s - kk * (BN / 4)) * 4;
        const int krow = k0 + kk;
        int src = -1;
        if (krow < K) src = perm_c >= 0 ? (krow < perm_c ? krow + 3 : krow - perm_c) : krow;
        const int col = n0 + c4;
        float* dst = Ws + kk * BN + c4;
        if (src >= 0 && row_aligned && col + 3 < N) {
            cp_async16(dst, W + (size_t)src * N + col);
        } else {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (src >= 0) {
                const float* p = W + (size_t)src * N + col;
                if (col + 0 < N) v.x = __ldg(p + 0);
                if (col + 1 < N) v.y = __ldg(p + 1);
                if (col + 2 < N) v.z = __ldg(p + 2);
                if (col + 3 < N) v.w = __ldg(p + 3);
            }
            *reinterpret_cast<float4*>(dst) = v;
        }
    }
}

// acc[8][TN] += A[rows ty*8..+8][0..kcount) * Ws[0..kcount)[cols]   (thread cols: tx*4..+3 and, TN==8, 64+tx*4..+3)
template <int TN>
__device__ __forceinline__ void mma_chunk(const float* a_base, int lda, const float* Ws, int kcount,
                                          float (&acc)[8][TN], int ty, int tx) {
    constexpr int BN = 16 * TN;
    const float* arow = a_base + (size_t)(ty * 8) * lda;
    for (int kk = 0; kk < kcount; kk += 4) {
        float4 a[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = *reinterpret_cast<const float4*>(arow + (size_t)i * lda + kk);
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
            const float4 b0 = *reinterpret_cast<const float4*>(Ws + (kk + k4) * BN + tx * 4);
            float4 b1 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (TN == 8) b1 = *reinterpret_cast<const float4*>(Ws + (kk + k4) * BN + 64 + tx * 4);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float av = k4 == 0 ? a[i].x : (k4 == 1 ? a[i].y : (k4 == 2 ? a[i].z : a[i].w));
                acc[i][0] = fmaf(av, b0.x, acc[i][0]);
                acc[i][1] = fmaf(av, b0.y, acc[i][1]);
                acc[i][2] = fmaf(av, b0.z, acc[i][2]);
                acc[i][3] = fmaf(av, b0.w, acc[i][3]);
                if (TN == 8) {
                    acc[i][4] = fmaf(av, b1.x, acc[i][4]);
                    acc[i][5] = fmaf(av, b1.y, acc[i][5]);
                    acc[i][6] = fmaf(av, b1.z, acc[i][6]);
                    acc[i][7] = fmaf(av, b1.w, acc[i][7]);
                }
            }
        }
    }
}

// Full K loop of one (tile, n0) output block: acc = A[BM][K4] . W[:, n0:n0+BN], A resident in shared memory.
template <int TN>
__device__ __forceinline__ void gemm_smemA(const float* A, int lda, int K, const float* __restrict__ W, int N, int n0,
                                           int perm_c, float* Ws /* 2*BK*BN_MAX */, float (&acc)[8][TN], int tid) {
    constexpr int BN = 16 * TN;
    const int ty = tid >> 4, tx = tid & 15;
    const int K4 = (K + 3) & ~3;
    const int nchunks = (K4 + BK - 1) / BK;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
    load_w_chunk<BN>(Ws, W, K, N, 0, n0, perm_c, tid);
    cp_async_commit();
    for (int c = 0; c < nchunks; ++c) {
        float* cur = Ws + (c & 1) * (BK * BN_MAX);
        if (c + 1 < nchunks) {
            load_w_chunk<BN>(Ws + ((c + 1) & 1) * (BK * BN_MAX), W, K, N, (c + 1) * BK, n0, perm_c, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const int kc = min(BK, K4 - c * BK);
        mma_chunk<TN>(A + c * BK, lda, cur, kc, acc, ty, tx);
        __syncthreads();
    }
}

struct TileInfo {
    long long g0;     // first group of the tile
    int ngroups;      // groups in this tile
    int rows;         // ngroups * K
};

// scale/shift/ReLU epilogue of an inner layer: write the thread's 8 x TN block into the next activation buffer
template <int TN>
__device__ __forceinline__ void store_inner(const float (&acc)[8][TN], float* out, int ldo, int n0, int N,
                                            const float* __restrict__ scale, const float* __restrict__ shift,
                                            int relu, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
#pragma unroll
    for (int h = 0; h < TN / 4; ++h) {
        const int col = n0 + h * 64 + tx * 4;
        if (col >= N) continue;
        float sc[4], sh[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const bool ok = col + j < N;
            sc[j] = ok ? (scale ? __ldg(scale + col + j) : 1.f) : 0.f;
            sh[j] = ok ? __ldg(shift + col + j) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float4 v;
            v.x = fmaf(acc[i][h * 4 + 0], sc[0], sh[0]);
            v.y = fmaf(acc[i][h * 4 + 1], sc[1], sh[1]);
            v.z = fmaf(acc[i][h * 4 + 2], sc[2], sh[2]);
            v.w = fmaf(acc[i][h * 4 + 3], sc[3], sh[3]);
            if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            *reinterpret_cast<float4*>(out + (size_t)(ty * 8 + i) * ldo + col) = v;   // pad cols get 0*.. = shift 0
        }
    }
}

// Last layer: scale/shift/ReLU then either direct row store (K == 1) or max over each run of K rows.
template <int TN>
__device__ __forceinline__ void store_last(const float (&acc)[8][TN], int n0, int N, const float* __restrict__ scale,
                                           const float* __restrict__ shift, int relu, int K, const TileInfo& ti,
                                           int* s_pool /* [BM][BN_MAX] worst case G=BM.. sized G*BN */,
                                           float* __restrict__ out, int tid) {
    constexpr int BN = 16 * TN;
    const int ty = tid >> 4, tx = tid & 15;
    if (K > 1) {
        for (int s = tid; s < ti.ngroups * BN; s += kMlpThreads) s_pool[s] = f2ord(__int_as_float(0xff800000));   // -inf
        __syncthreads();
    }
#pragma unroll
    for (int h = 0; h < TN / 4; ++h) {
        const int col = n0 + h * 64 + tx * 4;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (col + j >= N) continue;
            const float sc = scale ? __ldg(scale + col + j) : 1.f;
            const float sh = __ldg(shift + col + j);
            if (K == 1) {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int row = ty * 8 + i;
                    if (row < ti.rows) {
                        float v = fmaf(acc[i][h * 4 + j], sc, sh);
                        if (relu) v = fmaxf(v, 0.f);
                        out[(size_t)(ti.g0 + row) * N + col + j] = v;
                    }
                }
            } else {
                int curg = -1;
                float m = 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int row = ty * 8 + i;
                    if (row >= ti.rows) break;
                    float v = fmaf(acc[i][h * 4 + j], sc, sh);
                    if (relu) v = fmaxf(v, 0.f);
                    const int g = row / K;
                    if (g != curg) {
                        if (curg >= 0) atomicMax(&s_pool[curg * BN + h * 64 + tx * 4 + j], f2ord(m));
                        curg = g;
                        m = v;
                    } else {
                        m = fmaxf(m, v);
                    }
                }
                if (curg >= 0) atomicMax(&s_pool[curg * BN + h * 64 + tx * 4 + j], f2ord(m));
            }
        }
    }
    if (K > 1) {
        __syncthreads();
        for (int s = tid; s < ti.ngroups * BN; s += kMlpThreads) {
            const int g = s / BN, cl = s - g * BN;
            if (n0 + cl < N) out[(size_t)(ti.g0 + g) * N + n0 + cl] = ord2f(s_pool[s]);
        }
        __syncthreads();
    }
}

enum GatherMode { kGatherSA = 0, kGatherEdge = 1 };

struct FusedArgs {
    psa_mlp mlp;
    // geometry
    long long groups;     // total neighbourhoods (b*m for SA, b*n for EdgeConv)
    int K;                // rows per neighbourhood (nsample / k)
    int G;                // neighbourhoods per tile
    int n;                // dataset points per cloud
    int m;                // queries per cloud (SA) or n (EdgeConv)
    int c;                // feature channels per point
    int ldX, ldY;         // activation buffer leading dimensions (floats, multiples of 4)
    const float* xyz;     // SA: (b,n,3)
    const float* new_xyz; // SA: (b,m,3)
    const float* feat;    // SA: points (b,n,c) ; Edge: x (b,n,c)
    const int* idx;       // (groups, K)
    float* out;           // (groups, C_L)
};

template <int MODE>
__device__ __forceinline__ void gather_tile(const FusedArgs& a, const TileInfo& ti, float* X, int tid) {
    const int lane = tid & 31, warp = tid >> 5;
    const int C0 = a.mlp.channels[0];
    const int C04 = (C0 + 3) & ~3;
    const int c = a.c;
    for (int r = warp; r < BM; r += kMlpThreads / 32) {
        float* xr = X + (size_t)r * a.ldX;
        if (r >= ti.rows) {
            for (int l = lane; l < C04; l += 32) xr[l] = 0.f;
            continue;
        }
        const long long gid = ti.g0 + r / a.K;
        const long long bi = gid / a.m;
        const int j = __ldg(a.idx + gid * a.K + (r % a.K));
        if (MODE == kGatherSA) {
            if (c > 0) {
                const float* src = a.feat + ((size_t)bi * a.n + j) * c;
                if ((c & 3) == 0 && (reinterpret_cast<uintptr_t>(a.feat) & 15) == 0) {
                    for (int l = lane * 4; l < c; l += 128) cp_async16(xr + l, src + l);
                } else {
                    for (int l = lane; l < c; l += 32) xr[l] = __ldg(src + l);
                }
            }
            if (lane < 3) {
                // grouped_xyz - new_xyz (pointnet_util.py:46)
                xr[c + lane] = __ldg(a.xyz + ((size_t)bi * a.n + j) * 3 + lane) - __ldg(a.new_xyz + gid * 3 + lane);
            } else if (c + lane < C04) {
                xr[c + lane] = 0.f;
            }
        } else {
            // [x_i, x_j - x_i] (dgcnn/utils/tf_util.py:705)
            const float* ctr = a.feat + (size_t)gid * c;
            const float* nb = a.feat + ((size_t)bi * a.n + j) * c;
            for (int l = lane; l < c; l += 32) {
                const float ci = __ldg(ctr + l);
                xr[l] = ci;
                xr[c + l] = __ldg(nb + l) - ci;
            }
            for (int l = 2 * c + lane; l < C04; l += 32) xr[l] = 0.f;
        }
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
}

template <int MODE>
__global__ void __launch_bounds__(kMlpThreads, 1)
fused_group_mlp_kernel(const __grid_constant__ FusedArgs a) {
    extern __shared__ __align__(16) float smem_f[];
    float* X = smem_f;
    float* Y = X + (size_t)BM * a.ldX;
    float* Ws = Y + (size_t)BM * a.ldY;                       // 2 * BK * BN_MAX
    int* s_pool = reinterpret_cast<int*>(Ws + 2 * BK * BN_MAX);   // G * BN_MAX
    const int tid = threadIdx.x;
    const int L = a.mlp.n_layers;
    const long long ntiles = (a.groups + a.G - 1) / a.G;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        TileInfo ti;
        ti.g0 = t * a.G;
        ti.ngroups = (int)min((long long)a.G, a.groups - ti.g0);
        ti.rows = ti.ngroups * a.K;
        gather_tile<MODE>(a, ti, X, tid);
        for (int l = 0; l < L; ++l) {
            const int Cin = a.mlp.channels[l], Cout = a.mlp.channels[l + 1];
            const float* in = (l & 1) ? Y : X;
            float* outb = (l & 1) ? X : Y;
            const int ldi = (l & 1) ? a.ldY : a.ldX;
            const int ldo = (l & 1) ? a.ldX : a.ldY;
            const int perm_c = (MODE == kGatherSA && l == 0 && a.c > 0) ? a.c : -1;
            const bool last = (l == L - 1);
            const float* W = a.mlp.weight[l];
            const float* sc = a.mlp.scale[l];
            const float* sh = a.mlp.shift[l];
            const int relu = a.mlp.relu[l];
            if ((Cout % 128) == 0 || Cout > 64) {
                for (int n0 = 0; n0 < Cout; n0 += 128) {
                    float acc[8][8];
                    gemm_smemA<8>(in, ldi, Cin, W, Cout, n0, perm_c, Ws, acc, tid);
                    if (!last) store_inner<8>(acc, outb, ldo, n0, Cout, sc, sh, relu, tid);
                    else store_last<8>(acc, n0, Cout, sc, sh, relu, a.K, ti, s_pool, a.out, tid);
                }
            } else {
                for (int n0 = 0; n0 < Cout; n0 += 64) {
                    float acc[8][4];
                    gemm_smemA<4>(in, ldi, Cin, W, Cout, n0, perm_c, Ws, acc, tid);
                    if (!last) store_inner<4>(acc, outb, ldo, n0, Cout, sc, sh, relu, tid);
                    else store_last<4>(acc, n0, Cout, sc, sh, relu, a.K, ti, s_pool, a.out, tid);
                }
            }
            if (!last) {
                // zero the k-padding columns [Cout, round4(Cout)) of the buffer just written
                const int C4 = (Cout + 3) & ~3;
                if (C4 != Cout)
                    for (int s = tid; s < BM * (C4 - Cout); s += kMlpThreads)
                        outb[(size_t)(s / (C4 - Cout)) * ldo + Cout + s % (C4 - Cout)] = 0.f;
                __syncthreads();
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------------------
// Dense single layer: out = relu?((x . W [+ group_add[r / group_rows]] [+ xyz3[r] . w3]) * scale + shift) with optional max over
// runs of pool_k rows.
// A streamed from global in [BM][BK] chunks (cp.async when the row pitch allows 16-byte copies).
// ------------------------------------------------------------------------------------------------------------
constexpr int LDA_D = BK + 4;   // 20 floats = 80 B rows: 16-byte aligned, conflict-light

__device__ __forceinline__ void load_a_chunk(float* As, const float* __restrict__ x, long long row0, long long rows,
                                             int K, int k0, int tid) {
    const bool aligned = ((K & 3) == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
#pragma unroll
    for (int s = tid; s < BM * (BK / 4); s += kMlpThreads) {
        const int r = s / (BK / 4);
        const int k4 = (s - r * (BK / 4)) * 4;
        float* dst = As + r * LDA_D + k4;
        const long long row = row0 + r;
        const int k = k0 + k4;
        if (row < rows && aligned && k + 3 < K) {
            cp_async16(dst, x + row * K + k);
        } else {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (row < rows) {
                const float* p = x + row * K + k;
                if (k + 0 < K) v.x = __ldg(p + 0);
                if (k + 1 < K) v.y = __ldg(p + 1);
                if (k + 2 < K) v.z = __ldg(p + 2);
                if (k + 3 < K) v.w = __ldg(p + 3);
            }
            *reinterpret_cast<float4*>(dst) = v;
        }
    }
}

template <int TN>
__global__ void __launch_bounds__(kMlpThreads, 2)
dense_layer_kernel(const __grid_constant__ DenseArgs a) {
    constexpr int BN = 16 * TN;
    __shared__ __align__(16) float As[2][BM * LDA_D];
    __shared__ __align__(16) float Ws[2][BK * BN];
    __shared__ int s_pool[(TN == 8) ? 16 * BN : 32 * BN];   // pooled groups per tile: BM/pool_k <= this / BN
    const int tid = threadIdx.x;
    const int ty = tid >> 4, tx = tid & 15;
    const long long row0 = (long long)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int K4 = (a.K + 3) & ~3;
    const int nchunks = (K4 + BK - 1) / BK;
    float acc[8][TN];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
    load_a_chunk(As[0], a.x, row0, a.rows, a.K, 0, tid);
    load_w_chunk<BN>(Ws[0], a.W, a.K, a.N, 0, n0, -1, tid);
    cp_async_commit();
    for (int c = 0; c < nchunks; ++c) {
        if (c + 1 < nchunks) {
            load_a_chunk(As[(c + 1) & 1], a.x, row0, a.rows, a.K, (c + 1) * BK, tid);
            load_w_chunk<BN>(Ws[(c + 1) & 1], a.W, a.K, a.N, (c + 1) * BK, n0, -1, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        mma_chunk<TN>(As[c & 1], LDA_D, Ws[c & 1], min(BK, K4 - c * BK), acc, ty, tx);
        __syncthreads();
    }
    const int tile_rows = (int)min((long long)BM, a.rows - row0);
    const int pk = a.pool_k;
    if (a.group_add != nullptr) {      // the per-group input (pool_k == 1), in a pass of its own: the epilogue is the same code without it
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int row = ty * 8 + i;
            if (row >= tile_rows) break;
            const float* ga = a.group_add + (row0 + row) / a.group_rows * a.N;
#pragma unroll
            for (int h = 0; h < TN / 4; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int col = n0 + h * 64 + tx * 4 + j;
                    if (col < a.N) acc[i][h * 4 + j] += __ldg(ga + col);
                }
        }
    }
    if (a.xyz3 != nullptr) {           // the side input (pool_k == 1), in the same order as tc_dense_kernel's epilogue
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int row = ty * 8 + i;
            if (row >= tile_rows) break;
            const float* q = a.xyz3 + (row0 + row) * 3;
            const float x0 = __ldg(q), x1 = __ldg(q + 1), x2 = __ldg(q + 2);
#pragma unroll
            for (int h = 0; h < TN / 4; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int col = n0 + h * 64 + tx * 4 + j;
                    if (col < a.N)
                        acc[i][h * 4 + j] = fmaf(x2, __ldg(a.w3 + 2 * a.N + col), fmaf(x1, __ldg(a.w3 + a.N + col), fmaf(x0, __ldg(a.w3 + col), acc[i][h * 4 + j])));
                }
        }
    }
    if (pk == 1) {
#pragma unroll
        for (int h = 0; h < TN / 4; ++h) {
            const int col = n0 + h * 64 + tx * 4;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (col + j >= a.N) continue;
                const float sc = a.scale ? __ldg(a.scale + col + j) : 1.f;
                const float sh = a.shift ? __ldg(a.shift + col + j) : 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int row = ty * 8 + i;
                    if (row < tile_rows) {
                        float v = fmaf(acc[i][h * 4 + j], sc, sh);
                        if (a.relu) v = fmaxf(v, 0.f);
                        a.out[(row0 + row) * a.N + col + j] = v;
                    }
                }
            }
        }
        return;
    }
    // pooled: groups of pk consecutive rows.  pk <= BM and BM % pk == 0: groups live inside the tile -> shared
    // atomics then plain stores.  pk > BM (pk % BM == 0): the tile lies inside ONE group -> reduce in shared
    // memory, then one global atomicMax per column (out pre-filled with -inf by the launcher).
    const bool inside = pk <= BM;
    const int ngroups = inside ? (tile_rows / pk) : 1;
    for (int s = tid; s < ngroups * BN; s += kMlpThreads) s_pool[s] = f2ord(__int_as_float(0xff800000));
    __syncthreads();
#pragma unroll
    for (int h = 0; h < TN / 4; ++h) {
        const int col = n0 + h * 64 + tx * 4;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (col + j >= a.N) continue;
            const float sc = a.scale ? __ldg(a.scale + col + j) : 1.f;
            const float sh = a.shift ? __ldg(a.shift + col + j) : 0.f;
            int curg = -1;
            float m = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int row = ty * 8 + i;
                if (row >= tile_rows) break;
                float v = fmaf(acc[i][h * 4 + j], sc, sh);
                if (a.relu) v = fmaxf(v, 0.f);
                const int g = inside ? row / pk : 0;
                if (g != curg) {
                    if (curg >= 0) atomicMax(&s_pool[curg * BN + h * 64 + tx * 4 + j], f2ord(m));
                    curg = g;
                    m = v;
                } else {
                    m = fmaxf(m, v);
                }
            }
            if (curg >= 0) atomicMax(&s_pool[curg * BN + h * 64 + tx * 4 + j], f2ord(m));
        }
    }
    __syncthreads();
    for (int s = tid; s < ngroups * BN; s += kMlpThreads) {
        const int g = s / BN, cl = s - g * BN;
        if (n0 + cl >= a.N) continue;
        if (inside) {
            a.out[(row0 / pk + g) * a.N + n0 + cl] = ord2f(s_pool[s]);
        } else {
            atomicMax(reinterpret_cast<int*>(a.out) + (row0 / pk) * a.N + n0 + cl, s_pool[s]);
        }
    }
}


// ------------------------------------------------------------------------------------------------------------
// Small-M layer (rows <= 32: the FC heads, B = 32 rows x 1024 -> 512 -> 256 -> num_class).  The work is tiny and a
// single CTA per column block would be one long L2-latency chain, so K is split over the grid as well:
//   pass 1  CTA (col block of 32, k slice of 64): x slice staged transposed in shared memory, 4 warps x 16 k,
//           lane = output column (coalesced weight rows), 32 row-accumulators per thread, warps combined in shared
//           memory in fixed order, partial (32 x 32) written to the workspace;
//   pass 2  sums the K-slices in ascending order (deterministic) and applies scale / shift / ReLU.
// ------------------------------------------------------------------------------------------------------------
constexpr int kFcKs = 64;      // k per CTA
constexpr int kFcWarps = 4;

__global__ void __launch_bounds__(kFcWarps * 32)
fc_partial_kernel(const __grid_constant__ DenseArgs a, float* __restrict__ partial) {
    __shared__ float xs[kFcKs * 33];                  // [kk][r] padded: conflict-free transposed staging
    __shared__ float red[kFcWarps][32][33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int rows = (int)a.rows;
    const int ks = blockIdx.y, k0 = ks * kFcKs;
    const int kn = min(kFcKs, a.K - k0);
    for (int e0 = threadIdx.x; e0 < 32 * kFcKs; e0 += kFcWarps * 32 * 4) {
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int e = e0 + u * kFcWarps * 32;
            const int r = e / kFcKs, kk = e - r * kFcKs;
            v[u] = (e < 32 * kFcKs && r < rows && kk < kn) ? __ldg(a.x + (size_t)r * a.K + k0 + kk) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int e = e0 + u * kFcWarps * 32;
            if (e < 32 * kFcKs) { const int r = e / kFcKs, kk = e - r * kFcKs; xs[kk * 33 + r] = v[u]; }
        }
    }
    const int col = blockIdx.x * 32 + lane;
    constexpr int KW = kFcKs / kFcWarps;              // 16 k per warp
    float wv[KW];
#pragma unroll
    for (int u = 0; u < KW; ++u) {
        const int k = k0 + warp * KW + u;
        wv[u] = (col < a.N && k < a.K) ? __ldg(a.W + (size_t)k * a.N + col) : 0.f;
    }
    __syncthreads();
    float acc[32];
#pragma unroll
    for (int r = 0; r < 32; ++r) acc[r] = 0.f;
#pragma unroll
    for (int u = 0; u < KW; ++u) {
        const float* xr = xs + (warp * KW + u) * 33;
#pragma unroll
        for (int r = 0; r < 32; ++r) acc[r] = fmaf(xr[r], wv[u], acc[r]);
    }
#pragma unroll
    for (int r = 0; r < 32; ++r) red[warp][r][lane] = acc[r];
    __syncthreads();
    if (col < a.N)
        for (int r = warp; r < rows; r += kFcWarps) {
            float s = red[0][r][lane];
#pragma unroll
            for (int w = 1; w < kFcWarps; ++w) s += red[w][r][lane];
            partial[((size_t)ks * 32 + r) * a.N + col] = s;
        }
}

__global__ void fc_reduce_kernel(const __grid_constant__ DenseArgs a, const float* __restrict__ partial, int nks) {
    const int total = (int)a.rows * a.N;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
        const int r = e / a.N, col = e - r * a.N;
        float s = 0.f;
        for (int ks = 0; ks < nks; ++ks) s += partial[((size_t)ks * 32 + r) * a.N + col];
        float v = fmaf(s, a.scale ? __ldg(a.scale + col) : 1.f, a.shift ? __ldg(a.shift + col) : 0.f);
        if (a.relu) v = fmaxf(v, 0.f);
        a.out[e] = v;
    }
}

size_t fc_small_workspace_bytes(int K, int N) { return (size_t)((K + kFcKs - 1) / kFcKs) * 32 * N * sizeof(float); }

int launch_fc_small(const DenseArgs& d, float* partial, cudaStream_t st) {
    const int nks = (d.K + kFcKs - 1) / kFcKs;
    dim3 grid((d.N + 31) / 32, nks);
    fc_partial_kernel<<<grid, kFcWarps * 32, 0, st>>>(d, partial);
    const int total = (int)d.rows * d.N;
    fc_reduce_kernel<<<(total + 255) / 256, 256, 0, st>>>(d, partial, nks);
    return check_launch("fc_small");
}

__global__ void fill_ord_neg_inf_kernel(long long total, int* out, const unsigned int* run_if = nullptr) {
    if (run_if != nullptr && *run_if == 0u) return;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x)
        out[e] = f2ord(__int_as_float(0xff800000));
}
__global__ void decode_ord_kernel(long long total, int* out, const unsigned int* run_if = nullptr) {
    if (run_if != nullptr && *run_if == 0u) return;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x)
        out[e] = __float_as_int(ord2f(out[e]));
}

static int validate_mlp(const psa_mlp* mlp, const char* who) {
    PSA_REQUIRE(mlp != nullptr, "%s: null mlp", who);
    PSA_REQUIRE(mlp->n_layers >= 1 && mlp->n_layers <= PSA_MAX_MLP_LAYERS, "%s: n_layers=%d", who, mlp->n_layers);
    for (int l = 0; l <= mlp->n_layers; ++l)
        PSA_REQUIRE(mlp->channels[l] >= 1, "%s: channels[%d]=%d", who, l, mlp->channels[l]);
    for (int l = 0; l < mlp->n_layers; ++l)
        PSA_REQUIRE(mlp->weight[l] != nullptr && mlp->shift[l] != nullptr, "%s: layer %d has a null weight/shift", who, l);
    return PSA_OK;
}

int launch_dense(const DenseArgs& d, cudaStream_t st) {
    const long long tiles_m = (d.rows + BM - 1) / BM;
    PSA_SUPPORTED(tiles_m <= 0x7fffffffLL, "shared_mlp: too many rows");
    if (d.pool_k > 1) {
        PSA_SUPPORTED((d.pool_k >= 8 && d.pool_k <= BM && BM % d.pool_k == 0) || (d.pool_k % BM == 0),
                      "shared_mlp: pool_k=%d must divide %d (and be >= 8) or be a multiple of it", d.pool_k, BM);
        if (d.pool_k > BM) {
            long long total = d.rows / d.pool_k * d.N;
            fill_ord_neg_inf_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(total, reinterpret_cast<int*>(d.out));
        }
    }
    const bool wide = d.N > 64;
    if (wide) {
        dim3 grid((unsigned)tiles_m, (d.N + 127) / 128);
        dense_layer_kernel<8><<<grid, kMlpThreads, 0, st>>>(d);
    } else {
        dim3 grid((unsigned)tiles_m, (d.N + 63) / 64);
        dense_layer_kernel<4><<<grid, kMlpThreads, 0, st>>>(d);
    }
    if (d.pool_k > BM) {
        long long total = d.rows / d.pool_k * d.N;
        decode_ord_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(total, reinterpret_cast<int*>(d.out));
    }
    return check_launch("dense_layer_kernel");
}

template <int MODE>
static int launch_fused(FusedArgs& a, cudaStream_t st, const char* who) {
    const int L = a.mlp.n_layers;
    int maxX = 0, maxY = 0;
    for (int l = 0; l < L; ++l) {   // layer l reads buffer (l&1 ? Y : X)
        int c4 = (a.mlp.channels[l] + 3) & ~3;
        if (l & 1) maxY = max(maxY, c4); else maxX = max(maxX, c4);
    }
    a.ldX = maxX + 4;
    a.ldY = (maxY > 0 ? maxY : 0) + 4;
    a.G = a.K >= BM ? 1 : BM / a.K;
    PSA_SUPPORTED(a.K <= BM, "%s: nsample/k=%d exceeds the %d-row tile", who, a.K, BM);
    size_t smem = ((size_t)BM * (a.ldX + a.ldY) + 2 * BK * BN_MAX + (a.K > 1 ? (size_t)a.G * BN_MAX : 0)) * sizeof(float);
    PSA_SUPPORTED(smem <= 227 * 1024, "%s: MLP channel widths need %zu B of shared memory per tile (limit 227 KB)", who, smem);
    PSA_CUDA(cudaFuncSetAttribute(fused_group_mlp_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 1;
    PSA_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fused_group_mlp_kernel<MODE>, kMlpThreads, smem));
    if (occ < 1) occ = 1;
    const long long ntiles = (a.groups + a.G - 1) / a.G;
    long long grid = min(ntiles, (long long)kNumSMs * occ);
    fused_group_mlp_kernel<MODE><<<(int)grid, kMlpThreads, smem, st>>>(a);
    return check_launch("fused_group_mlp_kernel");
}

}  // namespace psa

using namespace psa;

namespace psa {
// fp32-FMA fused set-abstraction level (gather + MLP chain in shared memory + max-pool); idx already computed
int sa_module_simt(int b, int n, int m, int c, int nsample, const float* xyz, const float* new_xyz, const float* points,
                   const int* idx, const psa_mlp* mlp, float* out, cudaStream_t st) {
    FusedArgs a;
    a.mlp = *mlp;
    a.groups = (long long)b * m; a.K = nsample; a.n = n; a.m = m; a.c = c;
    a.xyz = xyz; a.new_xyz = new_xyz; a.feat = points; a.idx = idx; a.out = out;
    return launch_fused<kGatherSA>(a, st, "sa_module");
}
int validate_mlp_public(const psa_mlp* mlp, const char* who) { return validate_mlp(mlp, who); }
}  // namespace psa

namespace psa {
int edgeconv_simt(int b, int n, int c, int k, const float* x, const int* nn_idx, const psa_mlp* mlp, float* out, cudaStream_t st) {
    FusedArgs a;
    a.mlp = *mlp;
    a.groups = (long long)b * n; a.K = k; a.n = n; a.m = n; a.c = c;
    a.xyz = nullptr; a.new_xyz = nullptr; a.feat = x; a.idx = nn_idx; a.out = out;
    return launch_fused<kGatherEdge>(a, st, "edgeconv");
}
int launch_fill_ord_neg_inf(long long total, float* out, cudaStream_t st, const unsigned int* run_if) {
    fill_ord_neg_inf_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(total, reinterpret_cast<int*>(out), run_if);
    return check_launch("fill_ord_neg_inf_kernel");
}
int launch_decode_ord(long long total, float* out, cudaStream_t st, const unsigned int* run_if) {
    decode_ord_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(total, reinterpret_cast<int*>(out), run_if);
    return check_launch("decode_ord_kernel");
}
}  // namespace psa
