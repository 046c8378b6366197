// train_gemm.cuh -- the fp32 GEMM of the training path, with the layer's elementwise work fused into the operand loads.
//
// The reference trains through TF graph ops: conv2d (cuDNN) -> batch_norm (batch statistics) -> relu, each materialising a
// (B,m,K,C) tensor, and the mirrored gradient ops (pointnet2/utils/tf_util.py:155-185,512-531).  Here a level keeps ONE
// tensor per layer -- the PRE-batch-norm activations y_l -- and every other quantity is recomputed while tiles are staged:
//   ActIn   h_{l-1}[r][c] = relu(y_{l-1}[r][c] * scale[c] + shift[c]) (* dropout mask)      the forward input of layer l
//   GradIn  dy_l[r][c]    = ca[c] * dz + cb[c] * y_l[r][c] + cc[c],  dz = dh * [relu active]  the batch-norm backward
//           with dh either a dense tensor or the max-pool routing (dp[g][c] where argmax[g][c] == r mod K, else 0).
// Three products per layer, all on this kernel (C = A * B, fp32 FMA on float pairs, 128x128 / 128x64 / 64x64
// tiles, double-buffered shared memory, split over the contraction for the weight gradient):
//   forward          y_l  = ActIn   * W            A contraction-contiguous, B column-contiguous
//   input gradient   dh   = GradIn  * W^T          A contraction-contiguous, B contraction-contiguous
//   weight gradient  dW   = ActIn^T * GradIn       A row-contiguous (transposed read), B column-contiguous, split-K
// fp32 FMA keeps the gradients within the reference tests' 1e-4 (tf_grouping_op_test.py:25) without an operand split.
#pragma once
#include "common.cuh"

namespace psa {

struct ActIn : psa_act_in {   // fields: include/psa.h
    ActIn() = default;
    __host__ explicit ActIn(const psa_act_in& a) : psa_act_in(a) {}
    __device__ __forceinline__ float get(long long r, int c) const {
        float v = __ldg(x + r * ld + c);
        if (scale != nullptr) {
            v = fmaf(v, __ldg(scale + c), __ldg(shift + c));
            if (relu) v = fmaxf(v, 0.f);
        }
        if (mask != nullptr) v *= __ldg(mask + r * ld + c);
        return v;
    }
    __device__ __forceinline__ float4 get4(long long r, int c) const {
        float4 v = __ldg(reinterpret_cast<const float4*>(x + r * ld + c));
        if (scale != nullptr) {
            const float4 s = __ldg(reinterpret_cast<const float4*>(scale + c)), t = __ldg(reinterpret_cast<const float4*>(shift + c));
            v.x = fmaf(v.x, s.x, t.x); v.y = fmaf(v.y, s.y, t.y); v.z = fmaf(v.z, s.z, t.z); v.w = fmaf(v.w, s.w, t.w);
            if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        }
        if (mask != nullptr) {
            const float4 m = __ldg(reinterpret_cast<const float4*>(mask + r * ld + c));
            v.x *= m.x; v.y *= m.y; v.z *= m.z; v.w *= m.w;
        }
        return v;
    }
    __device__ __forceinline__ bool vec_ok() const {
        return (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (mask == nullptr || (reinterpret_cast<uintptr_t>(mask) & 15) == 0) &&
               (scale == nullptr || ((reinterpret_cast<uintptr_t>(scale) & 15) == 0 && (reinterpret_cast<uintptr_t>(shift) & 15) == 0));
    }
};

struct GradIn : psa_grad_in {   // fields: include/psa.h
    GradIn() = default;
    __host__ explicit GradIn(const psa_grad_in& g) : psa_grad_in(g) {}

    __device__ __forceinline__ float dz1(long long r, int c, float yv) const {
        float dz;
        if (mode == 0) {
            dz = __ldg(dh + r * ld_dh + c);
            if (mask != nullptr) dz *= __ldg(mask + r * ld_dh + c);
            if (s != nullptr && relu && !(fmaf(yv, __ldg(s + c), __ldg(t + c)) > 0.f)) dz = 0.f;
        } else {
            const long long g = r / pool_k;
            const int kk = (int)(r - g * pool_k);
            const size_t o = (size_t)g * C + c;
            dz = (__ldg(argk + o) == kk && __ldg(pv + o) > 0.f) ? __ldg(dp + o) : 0.f;
        }
        return dz;
    }
    __device__ __forceinline__ float get(long long r, int c) const {
        const float yv = (s != nullptr || ca != nullptr) ? __ldg(y + r * ld + c) : 0.f;
        const float dz = dz1(r, c, yv);
        if (ca == nullptr) return dz;
        return fmaf(__ldg(ca + c), dz, fmaf(__ldg(cb + c), yv, __ldg(cc + c)));
    }
    __device__ __forceinline__ float4 y4(long long r, int c) const {
        return (s != nullptr || ca != nullptr) ? __ldg(reinterpret_cast<const float4*>(y + r * ld + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    // dz = gradient w.r.t. the batch-norm OUTPUT of this layer (after the relu mask / pool routing / dropout)
    __device__ __forceinline__ float4 dz4(long long r, int c, const float4 yv) const {
        float4 dz;
        if (mode == 0) {
            dz = __ldg(reinterpret_cast<const float4*>(dh + r * ld_dh + c));
            if (mask != nullptr) {
                const float4 m = __ldg(reinterpret_cast<const float4*>(mask + r * ld_dh + c));
                dz.x *= m.x; dz.y *= m.y; dz.z *= m.z; dz.w *= m.w;
            }
            if (s != nullptr && relu) {
                const float4 s4 = __ldg(reinterpret_cast<const float4*>(s + c)), t4 = __ldg(reinterpret_cast<const float4*>(t + c));
                if (!(fmaf(yv.x, s4.x, t4.x) > 0.f)) dz.x = 0.f;
                if (!(fmaf(yv.y, s4.y, t4.y) > 0.f)) dz.y = 0.f;
                if (!(fmaf(yv.z, s4.z, t4.z) > 0.f)) dz.z = 0.f;
                if (!(fmaf(yv.w, s4.w, t4.w) > 0.f)) dz.w = 0.f;
            }
        } else {
            const long long g = r / pool_k;
            const int kk = (int)(r - g * pool_k);
            const size_t o = (size_t)g * C + c;
            const int4 a = __ldg(reinterpret_cast<const int4*>(argk + o));
            const float4 p = __ldg(reinterpret_cast<const float4*>(pv + o)), d = __ldg(reinterpret_cast<const float4*>(dp + o));
            dz.x = (a.x == kk && p.x > 0.f) ? d.x : 0.f;
            dz.y = (a.y == kk && p.y > 0.f) ? d.y : 0.f;
            dz.z = (a.z == kk && p.z > 0.f) ? d.z : 0.f;
            dz.w = (a.w == kk && p.w > 0.f) ? d.w : 0.f;
        }
        return dz;
    }
    __device__ __forceinline__ float4 get4(long long r, int c) const {
        const float4 yv = y4(r, c);
        const float4 dz = dz4(r, c, yv);
        if (ca == nullptr) return dz;
        const float4 a4 = __ldg(reinterpret_cast<const float4*>(ca + c)), b4 = __ldg(reinterpret_cast<const float4*>(cb + c));
        const float4 c4 = __ldg(reinterpret_cast<const float4*>(cc + c));
        return make_float4(fmaf(a4.x, dz.x, fmaf(b4.x, yv.x, c4.x)), fmaf(a4.y, dz.y, fmaf(b4.y, yv.y, c4.y)),
                           fmaf(a4.z, dz.z, fmaf(b4.z, yv.z, c4.z)), fmaf(a4.w, dz.w, fmaf(b4.w, yv.w, c4.w)));
    }
    __device__ __forceinline__ bool vec_ok() const {
        auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
        if (!al(y) || !al(s) || !al(t) || !al(ca) || !al(cb) || !al(cc)) return false;
        if ((s != nullptr || ca != nullptr) && (ld & 3) != 0) return false;
        if (mode == 0) return (ld_dh & 3) == 0 && al(dh) && al(mask);
        return (C & 3) == 0 && al(dp) && al(pv) && al(argk);
    }
};

// plain matrix operand (weights): element (r, c) = p[r * ld + c]
struct MatIn {
    const float* p;
    long long ld;
    __device__ __forceinline__ float get(long long r, int c) const { return __ldg(p + r * ld + c); }
    __device__ __forceinline__ float4 get4(long long r, int c) const { return __ldg(reinterpret_cast<const float4*>(p + r * ld + c)); }
    __device__ __forceinline__ bool vec_ok() const { return (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
};

constexpr int kGemmThreads = 256;
constexpr int kGemmBK = 16;

// Optional contraction skipping: an A functor that declares `static constexpr bool kSkipK = true` provides
//   long long next_k(long long k, long long k_end, long long m0, int bm)
// = the first contraction block start >= k (k is one; the result is k plus a multiple of kGemmBK, or k_end) whose block can hold a
// non-zero product for the tile's rows [m0, m0 + bm).  Every other functor runs every block, as before.
template <class F, class = void>
struct GemmSkipK { static constexpr bool value = false; };
template <class F>
struct GemmSkipK<F, decltype((void)F::kSkipK)> { static constexpr bool value = F::kSkipK; };

struct GemmOut {
    float* out;            // (M, ld_out) -- or split-K partials (splits, M, N) when splits > 1
    long long ld_out;
    const float* bias;     // per output column, or null
    int col_skip;          // output columns [0, col_skip) are dropped, column c lands at c - col_skip
    float* stat_partial;   // (tiles_m, 2, N) per-tile column sums / sums of squares of the stored values, or null
    // GROUP instantiations: output row m adds group_add[m / group_rows] (N) before the bias (a per-group input row, e.g. a
    // global feature's product tiled over a cloud's points)
    const float* group_add = nullptr;
    long long group_rows = 0;
};

// Operand conventions.  A is logically (M, Kc), B is (Kc, N).
//   A_KC  : functor indexed (row = m, col = kc), contiguous along kc.      !A_KC: functor indexed (row = kc, col = m).
//   B_NC  : functor indexed (row = kc, col = n), contiguous along n.       !B_NC: functor indexed (row = n, col = kc).
template <int BM, int BN, bool A_KC, bool B_NC, class FA, class FB, bool GROUP = false>
__global__ void __launch_bounds__(kGemmThreads, 2)
train_gemm_kernel(const FA fa, const FB fb, const GemmOut o, long long M, int N, long long Kc, long long k_per_split) {
    constexpr int TM = BM / 16, TN = BN / 16;                 // 8 or 4
    constexpr int LDA = BM + 4, LDB = BN + 4;
    constexpr int LA = BM * kGemmBK / 4 / kGemmThreads;       // float4 loads per thread per stage (2 or 1)
    constexpr int LB = BN * kGemmBK / 4 / kGemmThreads;
    __shared__ __align__(16) float As[2][kGemmBK][LDA];
    __shared__ __align__(16) float Bs[2][kGemmBK][LDB];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const long long m0 = (long long)blockIdx.y * BM;
    const int n0 = blockIdx.x * BN;
    const long long k_begin = (long long)blockIdx.z * k_per_split;
    const long long k_end = min(Kc, k_begin + k_per_split);
    const bool va = fa.vec_ok(), vb = fb.vec_ok();

    float4 ra[LA], rb[LB];
    auto fetch = [&](long long k0) {
#pragma unroll
        for (int i = 0; i < LA; ++i) {
            const int id = tid + i * kGemmThreads;
            long long r; int c; bool full, any;
            if (A_KC) {                                  // (m = id / 4, kc = (id % 4) * 4): four consecutive kc of one row
                const long long m = m0 + (id >> 2); const long long kc = k0 + (id & 3) * 4;
                r = m; c = (int)kc; any = m < M && kc < k_end; full = m < M && kc + 3 < k_end;
                if (any && full && va) ra[i] = fa.get4(r, c);
                else {
                    float v[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) v[u] = (m < M && kc + u < k_end) ? fa.get(r, c + u) : 0.f;
                    ra[i] = make_float4(v[0], v[1], v[2], v[3]);
                }
            } else {                                     // (kc = id / (BM/4), m = (id % (BM/4)) * 4): four consecutive m of one kc
                const long long kc = k0 + id / (BM / 4); const long long m = m0 + (id % (BM / 4)) * 4;
                r = kc; c = (int)m; any = kc < k_end && m < M; full = kc < k_end && m + 3 < M;
                if (any && full && va) ra[i] = fa.get4(r, c);
                else {
                    float v[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) v[u] = (kc < k_end && m + u < M) ? fa.get(r, c + u) : 0.f;
                    ra[i] = make_float4(v[0], v[1], v[2], v[3]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < LB; ++i) {
            const int id = tid + i * kGemmThreads;
            if (B_NC) {
                const long long kc = k0 + id / (BN / 4); const int n = n0 + (id % (BN / 4)) * 4;
                if (kc < k_end && n + 3 < N && vb) rb[i] = fb.get4(kc, n);
                else {
                    float v[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) v[u] = (kc < k_end && n + u < N) ? fb.get(kc, n + u) : 0.f;
                    rb[i] = make_float4(v[0], v[1], v[2], v[3]);
                }
            } else {
                const int n = n0 + (id >> 2); const long long kc = k0 + (id & 3) * 4;
                if (n < N && kc + 3 < k_end && vb) rb[i] = fb.get4(n, (int)kc);
                else {
                    float v[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) v[u] = (n < N && kc + u < k_end) ? fb.get(n, (int)kc + u) : 0.f;
                    rb[i] = make_float4(v[0], v[1], v[2], v[3]);
                }
            }
        }
    };
    auto stash = [&](int buf) {
#pragma unroll
        for (int i = 0; i < LA; ++i) {
            const int id = tid + i * kGemmThreads;
            if (A_KC) {
                const int m = id >> 2, kc = (id & 3) * 4;
                As[buf][kc][m] = ra[i].x; As[buf][kc + 1][m] = ra[i].y; As[buf][kc + 2][m] = ra[i].z; As[buf][kc + 3][m] = ra[i].w;
            } else {
                const int kc = id / (BM / 4), m = (id % (BM / 4)) * 4;
                *reinterpret_cast<float4*>(&As[buf][kc][m]) = ra[i];
            }
        }
#pragma unroll
        for (int i = 0; i < LB; ++i) {
            const int id = tid + i * kGemmThreads;
            if (B_NC) {
                const int kc = id / (BN / 4), n = (id % (BN / 4)) * 4;
                *reinterpret_cast<float4*>(&Bs[buf][kc][n]) = rb[i];
            } else {
                const int n = id >> 2, kc = (id & 3) * 4;
                Bs[buf][kc][n] = rb[i].x; Bs[buf][kc + 1][n] = rb[i].y; Bs[buf][kc + 2][n] = rb[i].z; Bs[buf][kc + 3][n] = rb[i].w;
            }
        }
    };

    // thread (ty, tx): rows {ty*4 .. +4} (+ BM/2 for the second half when TM == 8), columns likewise
    float2 acc[TM][TN / 2];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN / 2; ++j) acc[i][j] = make_float2(0.f, 0.f);

    long long k_first = k_begin;
    if constexpr (GemmSkipK<FA>::value) {
        if (k_begin < k_end) k_first = fa.next_k(k_begin, k_end, m0, BM);
    }
    if (k_first < k_end) {
        fetch(k_first);
        stash(0);
        __syncthreads();
        int buf = 0;
        for (long long k0 = k_first, kn; k0 < k_end; k0 = kn) {
            kn = k0 + kGemmBK;
            if constexpr (GemmSkipK<FA>::value) {
                if (kn < k_end) kn = fa.next_k(kn, k_end, m0, BM);
            }
            const bool more = kn < k_end;
            if (more) fetch(kn);
#pragma unroll
            for (int kk = 0; kk < kGemmBK; ++kk) {
                float a[TM];
                float2 b[TN / 2];
                {
                    const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
                    a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
                    if (TM == 8) {
                        const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][BM / 2 + ty * 4]);
                        a[TM - 4] = a1.x; a[TM - 3] = a1.y; a[TM - 2] = a1.z; a[TM - 1] = a1.w;
                    }
                    const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
                    b[0] = make_float2(b0.x, b0.y); b[1] = make_float2(b0.z, b0.w);
                    if (TN == 8) {
                        const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][BN / 2 + tx * 4]);
                        b[TN / 2 - 2] = make_float2(b1.x, b1.y); b[TN / 2 - 1] = make_float2(b1.z, b1.w);
                    }
                }
#pragma unroll
                for (int i = 0; i < TM; ++i)
#pragma unroll
                    for (int j = 0; j < TN / 2; ++j) acc[i][j] = ffma2_rn(make_float2(a[i], a[i]), b[j], acc[i][j]);
            }
            if (more) {
                stash(buf ^ 1);
                __syncthreads();
                buf ^= 1;
            }
        }
    }

    // ---- epilogue ----
    float* outp = o.out + (gridDim.z > 1 ? (size_t)blockIdx.z * (size_t)M * (size_t)o.ld_out : 0);
    float csum[TN], csq[TN];
#pragma unroll
    for (int j = 0; j < TN; ++j) csum[j] = csq[j] = 0.f;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const long long m = m0 + ((TM == 8 && i >= 4) ? BM / 2 + ty * 4 + (i - 4) : ty * 4 + i);
#pragma unroll
        for (int jh = 0; jh < TN / 4; ++jh) {
            const int n = n0 + (jh == 1 ? BN / 2 : 0) + tx * 4;
            float v[4] = {acc[i][jh * 2].x, acc[i][jh * 2].y, acc[i][jh * 2 + 1].x, acc[i][jh * 2 + 1].y};
            if constexpr (GROUP) {
                if (m < M) {
                    const float* ga = o.group_add + (size_t)(m / o.group_rows) * N;
#pragma unroll
                    for (int u = 0; u < 4; ++u) if (n + u < N) v[u] += __ldg(ga + n + u);
                }
            }
            if (o.bias != nullptr) {
#pragma unroll
                for (int u = 0; u < 4; ++u) if (n + u < N) v[u] += __ldg(o.bias + n + u);
            }
            if (m < M) {
#pragma unroll
                for (int u = 0; u < 4; ++u) { csum[jh * 4 + u] += v[u]; csq[jh * 4 + u] = fmaf(v[u], v[u], csq[jh * 4 + u]); }
                float* dst = outp + (size_t)m * o.ld_out + (n - o.col_skip);
                if (n + 3 < N && n >= o.col_skip && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
                    *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
                } else {
#pragma unroll
                    for (int u = 0; u < 4; ++u) if (n + u < N && n + u >= o.col_skip) dst[u] = v[u];
                }
            }
        }
    }
    if (o.stat_partial != nullptr) {
        // column sums over the tile's rows: the 16 row-threads of a column fold through shared memory in ty order
        __syncthreads();
        float* red = &As[0][0][0];                           // 16 x BN x 2 floats <= 2*16*(BM+4) floats for BN <= BM
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int col = (j >= 4 ? BN / 2 : 0) + tx * 4 + (j & 3);
            red[(ty * BN + col) * 2] = csum[j];
            red[(ty * BN + col) * 2 + 1] = csq[j];
        }
        __syncthreads();
        for (int e = tid; e < BN * 2; e += kGemmThreads) {
            const int col = e >> 1, which = e & 1;
            float t = 0.f;
#pragma unroll
            for (int r = 0; r < 16; ++r) t += red[(r * BN + col) * 2 + which];
            if (n0 + col < N) o.stat_partial[((size_t)blockIdx.y * 2 + which) * N + n0 + col] = t;
        }
    }
}

}  // namespace psa
