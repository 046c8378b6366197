// spider.cu -- SpiderCNN's spiderConv layer (SpiderCNN/utils/tf_util.py:127-235), its group norm and its top-k pooling, inference.
//
// What the reference does per layer: group_point -> (B,N,k,C) neighbour features, 20 tiled (B,N,k,T) Taylor weights -> the filter
// g_t(delta) per neighbour slot, the product (B,N,k,C,T) reshaped to (B,N,k,C*T) with channel index c*T + t, then a [1,k] VALID
// conv2d (weights differ per slot j) + bias, group norm, ReLU.  At B=32, N=1024 the conv input of the last layer alone is 1.68 GB.
// What happens here:
//   spider_taylor_kernel   g (B*N*k, T) = the filter values, once per layer (13 MB at B=32, N=1024, k=20)
//   tc_spider_kernel       the conv as ONE GEMM over the B*N points, y = A . Wp + bias, whose A operand
//                          A[p][(j, t, c)] = h[nn(p,j)][c] * g[p][j][t] is never stored: the producer warps gather the rows h[nn(p,j)]
//                          of a 64-wide K block into shared memory, the consumers apply the previous layer's group norm (a per-cloud
//                          affine) + ReLU and the factor g while they split the block into tensor-core operands.  The weight rows
//                          are permuted to (j, t, c) order when the image is built, so a K block is one (j, t) slice of a
//                          gathered row (two for c = 32).  Runs on the shared ring (ring_gemm.cuh).
//   spider_fma_kernel      the same product on the fp32 FMA pipe (mode 1, and shapes the tensor path does not take: layer 1, c = 3)
//   group_norm_*           per (cloud, group) mean and centred variance in fp64 -> the per-cloud affine (scale, shift)
//   topk_pool_kernel       the two largest values of relu(y * scale + shift) per (cloud, channel)
// and the training backward of all of these (below the launchers of the forward).
#include <float.h>
#include <limits.h>

#include "common.cuh"
#include "ring_gemm.cuh"
#include "train_gemm.cuh"

namespace psa {

using namespace tc;

constexpr int kSpiderMaxK = 32;          // neighbour slots staged per tile row (shared memory)
constexpr int kTaylorTerms = 20;

// ------------------------------------------------------------------------------------------------------------------
// g[(p*k + j)*T + t] = sum_m taylor[m][t] mono_m(delta[p][j]), grouped as the reference sums it (tf_util.py:211-217)
// ------------------------------------------------------------------------------------------------------------------
__global__ void spider_taylor_kernel(long long pairs, int T, const float* __restrict__ delta, const float* __restrict__ taylor,
                                     float* __restrict__ g) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= pairs * T) return;
    const long long pj = e / T;
    const int t = (int)(e - pj * T);
    const float X = __ldg(delta + pj * 3), Y = __ldg(delta + pj * 3 + 1), Z = __ldg(delta + pj * 3 + 2);
    float w[kTaylorTerms];
#pragma unroll
    for (int m = 0; m < kTaylorTerms; ++m) w[m] = __ldg(taylor + m * T + t);
    // x, y, z, xyz, xy, yz, xz, 1, xx, yy, zz, xxy, xyy, xxz, xzz, yyz, yzz, xxx, yyy, zzz
    const float g1 = w[0] * X + w[1] * Y + w[2] * Z + w[3] * X * Y * Z;
    const float g2 = w[4] * X * Y + w[5] * Y * Z + w[6] * X * Z + w[7];
    const float g3 = w[8] * X * X + w[9] * Y * Y + w[10] * Z * Z;
    const float g4 = w[11] * X * X * Y + w[12] * X * Y * Y + w[13] * X * X * Z;
    const float g5 = w[14] * X * Z * Z + w[15] * Y * Y * Z + w[16] * Y * Z * Z;
    const float g6 = w[17] * X * X * X + w[18] * Y * Y * Y + w[19] * Z * Z * Z;
    g[e] = g1 + g2 + g3 + g4 + g5 + g6;
}

// W (k, c*T, N) in the reference's row order j*(c*T) + c*T + t -> Wp (k*T*c, N) in row order (j*T + t)*c + c
__global__ void spider_permute_kernel(int k, int c, int T, int N, const float* __restrict__ W, float* __restrict__ Wp) {
    const long long total = (long long)k * c * T * N;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int o = (int)(e % N);
        const long long row = e / N;                 // (j*T + t)*c + ch
        const int ch = (int)(row % c);
        const long long jt = row / c;
        const int t = (int)(jt % T), j = (int)(jt / T);
        Wp[e] = __ldg(W + (((long long)j * c + ch) * T + t) * N + o);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// tc_spider_kernel<NP, NC>: y (rows, N) = A . Wp + bias on the ring (ring_gemm.cuh), unit = 128-row tile x 64 NC-column tile, all
// K blocks.  Per unit a producer warp first copies its rows' k neighbour indices to shared memory, so the gathers of a block only
// wait on shared-memory reads.
// ------------------------------------------------------------------------------------------------------------------
struct SpiderArgs {
    long long rows;            // b * n
    int n, c, k, T, K, N;      // K = k * T * c, a multiple of 64 on the tensor path
    const float* feat;         // (rows, c), 16-byte aligned on the tensor path
    const int* idx;            // (rows, k)
    const float* g;            // (rows * k, T)
    const float* fs;           // (b, c) or null, 8-byte aligned on the tensor path
    const float* fu;
    const float* bias;         // (N), 8-byte aligned on the tensor path
    float* y;                  // (rows, N), 8-byte aligned on the tensor path
    RingArgs ring;             // Wp in the format of NP, tile width 64 NC
};

struct SpiderOp {
    const SpiderArgs& a;
    static constexpr bool kClaim = false;
    static constexpr uint32_t kBudget = kRingBudget;
    struct Smem {
        int nbr[128 * kSpiderMaxK];                        // the unit's neighbour rows (global row index)
    };
    struct Unit {
        int nb, col0;
        long long r[2];
        bool v[2];
        int cb[2];                                         // the rows' clouds
    };

    __device__ int units(int Nt) const { return (int)((a.rows + 127) / 128 * (a.N / Nt)); }

    template <class Put>
    __device__ void produce(int unit, int Nt, int pw, int lane, Smem& sm, Put&& put) const {
        const int NTC = a.N / Nt, KC = a.K / 64, seg = a.T * a.c;
        const long long row0 = (long long)(unit / NTC) * 128;
        const int nt = unit % NTC, r0 = 32 * pw, nr = (int)max(0LL, min(32LL, a.rows - row0 - r0));
        __syncwarp();                                      // the previous unit's reads of nbr are done
        for (int e = lane; e < nr * a.k; e += 32) {
            const int r = e / a.k;
            const long long p = row0 + r0 + r;
            sm.nbr[(r0 + r) * kSpiderMaxK + (e - r * a.k)] = (int)(p / a.n * a.n) + __ldg(a.idx + p * a.k + (e - r * a.k));
        }
        __syncwarp();
        for (int kb = 0; kb < KC; ++kb)
            put((size_t)nt * KC + kb, [&](uint32_t xs) {
                // lane (row half, 16-byte chunk): the chunk's column of the block is fixed per lane, so is its (j, t, c)
                const int cc = (lane & 15) * 4, kk = kb * 64 + cc;
                const int j = kk / seg, rem = kk - j * seg, ch = rem - rem / a.c * a.c;
                for (int r = lane >> 4; r < nr; r += 2) {
                    const int row = r0 + r;
                    cp_async16(xs + (uint32_t)row * kRingXRow + (uint32_t)cc * 4u, a.feat + (size_t)sm.nbr[row * kSpiderMaxK + j] * a.c + ch);
                }
            });
    }

    __device__ Unit unit(int unit, int Nt, int row, Smem&, int) const {
        const int NTC = a.N / Nt;
        Unit u;
        u.nb = a.K / 64;
        u.col0 = unit % NTC * Nt;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            u.r[i] = (long long)(unit / NTC) * 128 + row + 8 * i;
            u.v[i] = u.r[i] < a.rows;
            u.cb[i] = u.v[i] ? (int)(u.r[i] / a.n) * a.c : 0;
        }
        return u;
    }

    // the previous layer's group norm + ReLU, times g_t(delta_pj); rows past `rows` read as zero (their staged bytes are stale)
    __device__ void load(const Unit& u, const float* xs, int kb, int t, float2 (&x)[4][2][2]) const {
        const int seg = a.T * a.c;
        // c % 32 == 0: each 32-column half of the block lies in one (j, t) slice, channels ch0 ..
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int kk = kb * 64 + 32 * hf, j = kk / seg, rem = kk - j * seg, tt = rem / a.c, ch0 = rem - tt * a.c;
            float gv[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) gv[i] = u.v[i] ? __ldg(a.g + (u.r[i] * a.k + j) * a.T + tt) : 0.f;
#pragma unroll
            for (int s = 2 * hf; s < 2 * hf + 2; ++s)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int ch = ch0 + 16 * s + 8 * h + 2 * t - 32 * hf;
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        float2 v = make_float2(0.f, 0.f);
                        if (u.v[i]) {
                            v = staged_pair(xs, s, h, i, t);
                            if (a.fs != nullptr) {
                                const float2 sc = __ldg(reinterpret_cast<const float2*>(a.fs + u.cb[i] + ch));
                                const float2 sh = __ldg(reinterpret_cast<const float2*>(a.fu + u.cb[i] + ch));
                                v.x = fmaxf(fmaf(v.x, sc.x, sh.x), 0.f);
                                v.y = fmaxf(fmaf(v.y, sc.y, sh.y), 0.f);
                            }
                            v.x *= gv[i];
                            v.y *= gv[i];
                        }
                        x[s][h][i] = v;
                    }
                }
        }
    }

    // fp16x2 column factor, bias; pre-group-norm y
    __device__ void epilogue(const Unit& u, const float (&acc)[32], int col0, int t, const float* colscale, Smem&) const {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const int col = col0 + 8 * jj + 2 * t;
            const float2 cs = colscale != nullptr ? __ldg(reinterpret_cast<const float2*>(colscale + col)) : make_float2(1.f, 1.f);
            const float2 bi = __ldg(reinterpret_cast<const float2*>(a.bias + col));
#pragma unroll
            for (int i = 0; i < 2; ++i)
                if (u.v[i])
                    *reinterpret_cast<float2*>(a.y + (size_t)u.r[i] * a.N + col) =
                        make_float2(fmaf(acc[4 * jj + 2 * i], cs.x, bi.x), fmaf(acc[4 * jj + 2 * i + 1], cs.y, bi.y));
        }
    }

    // the FMA fallback's A, in the reference's K order (j, c, t)
    __device__ float load_a(long long p, int kk) const {
        const int ct = a.c * a.T, j = kk / ct, rem = kk - j * ct, ch = rem / a.T, tt = rem - ch * a.T;
        const int b = (int)(p / a.n);
        float x = __ldg(a.feat + ((long long)b * a.n + __ldg(a.idx + p * a.k + j)) * a.c + ch);
        if (a.fs != nullptr) x = fmaxf(fmaf(x, __ldg(a.fs + b * a.c + ch), __ldg(a.fu + b * a.c + ch)), 0.f);
        return x * __ldg(a.g + (p * a.k + j) * a.T + tt);
    }
    __device__ void store(long long p, int col, float s) const { a.y[(size_t)p * a.N + col] = s + __ldg(a.bias + col); }
};

template <int NP, int NC>
__global__ void __launch_bounds__(kRingThreads, 1) tc_spider_kernel(const __grid_constant__ SpiderArgs a) {
    ring_gemm<NP, NC>(SpiderOp{a}, a.ring);
}

// the same product on the fp32 FMA pipe, with the unpermuted W
__global__ void __launch_bounds__(256) spider_fma_kernel(const __grid_constant__ SpiderArgs a, const float* __restrict__ W) {
    fma_gemm(SpiderOp{a}, a.rows, a.K, a.N, W);
}

// ------------------------------------------------------------------------------------------------------------------
// Group norm as a per-cloud affine.  Block (group, cloud): the mean, then the centred sum of squares, both in fp64 and reduced
// in a fixed order.
// ------------------------------------------------------------------------------------------------------------------
__device__ double block_sum_256(double v, double* red) {
    const int tid = threadIdx.x;
    red[tid] = v;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (tid < w) red[tid] += red[tid + w];
        __syncthreads();
    }
    const double s = red[0];
    __syncthreads();
    return s;
}

__global__ void __launch_bounds__(256) group_norm_affine_kernel(int n, int c, int cpg, float eps, const float* __restrict__ y,
                                                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                float* __restrict__ scale, float* __restrict__ shift) {
    __shared__ double red[256];
    const int grp = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const long long cnt = (long long)n * cpg;
    const float* yb = y + (size_t)b * n * c + (size_t)grp * cpg;
    double s = 0.0;
    for (long long e = tid; e < cnt; e += 256) s += (double)__ldg(yb + (e / cpg) * c + e % cpg);
    const double mean = block_sum_256(s, red) / (double)cnt;
    double ss = 0.0;
    for (long long e = tid; e < cnt; e += 256) {
        const double d = (double)__ldg(yb + (e / cpg) * c + e % cpg) - mean;
        ss += d * d;
    }
    const double var = block_sum_256(ss, red) / (double)cnt;
    const double rstd = 1.0 / sqrt(var + (double)eps);
    for (int i = tid; i < cpg; i += 256) {
        const int ch = grp * cpg + i;
        const double sc = (double)__ldg(gamma + ch) * rstd;
        scale[(size_t)b * c + ch] = (float)sc;
        shift[(size_t)b * c + ch] = (float)((double)__ldg(beta + ch) - mean * sc);
    }
}

__global__ void cloud_affine_kernel(long long total, int n, int c, const float* __restrict__ y, const float* __restrict__ scale,
                                    const float* __restrict__ shift, int relu, float* __restrict__ out) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int ch = (int)(e % c);
        const long long bc = e / c / n * c + ch;
        float h = fmaf(__ldg(y + e), __ldg(scale + bc), __ldg(shift + bc));
        if (relu) h = fmaxf(h, 0.f);
        out[e] = h;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Top-2 over the points per (cloud, channel).  Block (32 channels, 8 point slices); the slices' pairs merged in slice order.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void top2_push(float v, float& m1, float& m2) {
    if (v > m1) { m2 = m1; m1 = v; }
    else if (v > m2) m2 = v;
}

__global__ void __launch_bounds__(256) topk_pool_kernel(int n, int c, const float* __restrict__ y, const float* __restrict__ scale,
                                                        const float* __restrict__ shift, int relu, float* __restrict__ out, int out_channels,
                                                        int offset) {
    __shared__ float s_top[8][32][2];
    const int tx = threadIdx.x, ty = threadIdx.y, b = blockIdx.y, ch = blockIdx.x * 32 + tx;
    float m1 = -INFINITY, m2 = -INFINITY;
    if (ch < c) {
        const float sc = scale ? __ldg(scale + (size_t)b * c + ch) : 1.f, sh = scale ? __ldg(shift + (size_t)b * c + ch) : 0.f;
        for (int p = ty; p < n; p += 8) {
            float h = __ldg(y + ((size_t)b * n + p) * c + ch);
            if (scale) h = fmaf(h, sc, sh);
            if (relu) h = fmaxf(h, 0.f);
            top2_push(h, m1, m2);
        }
    }
    s_top[ty][tx][0] = m1;
    s_top[ty][tx][1] = m2;
    __syncthreads();
    if (ty != 0 || ch >= c) return;
    for (int w = 1; w < 8; ++w) { top2_push(s_top[w][tx][0], m1, m2); top2_push(s_top[w][tx][1], m1, m2); }
    float* dst = out + ((size_t)b * out_channels + offset + ch) * 2;
    dst[0] = m1;
    dst[1] = m2;
}

// ------------------------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------------------------
// the shapes and pointers the tensor path takes: cp.async reads feat in 16-byte chunks, the split step reads feat_scale / feat_shift
// and the epilogue reads bias and writes y in float2.  A null pointer counts as aligned, so spider_ws sizes the workspace from the
// dims alone; a misaligned pointer sends the call to the FMA kernel, which reads and writes one float at a time.
static bool spider_tc_eligible(long long rows, int c, int k, int T, int N, const float* feat, const float* fs, const float* fu,
                               const float* bias, const float* y) {
    auto al = [](const void* p, uintptr_t m) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & m) == 0; };
    const long long K = (long long)k * T * c;
    return rows >= 128 && c % 32 == 0 && K % 64 == 0 && N >= 64 && N % 64 == 0 && (N == 64 || N % 128 == 0) && al(feat, 15) &&
           al(fs, 7) && al(fu, 7) && al(bias, 7) && al(y, 7);
}

struct SpiderWs {
    size_t g, wp, img2, img3, total;
};
static SpiderWs spider_ws(int b, int n, int c, int k, int T, int N) {
    SpiderWs w{};
    const long long rows = (long long)b * n;
    const int K = k * T * c;
    size_t off = 256;                                        // word 0: range flag of the fp16x2 launch
    w.g = off; off += al256((size_t)rows * k * T * sizeof(float));
    if (spider_tc_eligible(rows, c, k, T, N, nullptr, nullptr, nullptr, nullptr, nullptr)) {
        w.wp = off; off += al256((size_t)K * N * sizeof(float));
        w.img2 = off; off += tc_image_alloc_bytes(K, N, 2);
        w.img3 = off; off += tc_image_alloc_bytes(K, N, 3);
    }
    w.total = off;
    return w;
}

static const RingKernels kSpiderRing = {{{(const void*)tc_spider_kernel<2, 1>, (const void*)tc_spider_kernel<2, 2>},
                                         {(const void*)tc_spider_kernel<3, 1>, (const void*)tc_spider_kernel<3, 2>}},
                                        "tc_spider_kernel", SpiderOp::kBudget};

// ==================================================================================================================
// Training backward, fp32 FMA (train_gemm.cuh explains why fp32 FMA holds the 1e-4 gradient bound without an operand split).
// No float atomics: every sum runs in a fixed order, so a step is bit-reproducible.  Per layer, with dy the gradient of the
// pre-norm output y:
//   dW (k*c*T, N) = A^T . dy        train_gemm_kernel, A read through SpiderA (the forward's gathered operand, never stored)
//   D, dg                           spider_bwd_data_kernel: Q = dy . W^T per (64 points, slot j, channel chunk) in registers,
//                                   D[p][j][c] = sum_t g Q, dg[p][j][t] = sum_c h Q (chunks in order, then channel groups in order)
//   d taylor[m][t]                  spider_taylor_grad_kernel: sum over (p, j) of dg * mono_m(delta), fp64 block partials
//   dy of the layer below           spider_gn_bwd_kernel: top-2 routing + relu mask + group-norm backward per (group, cloud)
// ==================================================================================================================
constexpr int kTrainT = 5;               // Taylor channels compiled into the backward (SpiderCNN's taylor_channel)

// the forward's K operand in the reference's (j, c, t) row order, as train_gemm's transposed-read A (row = point, col = K row)
struct SpiderA {
    SpiderArgs a;
    __device__ __forceinline__ float get(long long p, int kk) const { return SpiderOp{a}.load_a(p, kk); }
    __device__ __forceinline__ float4 get4(long long p, int kk) const {
        const SpiderOp op{a};
        return make_float4(op.load_a(p, kk), op.load_a(p, kk + 1), op.load_a(p, kk + 2), op.load_a(p, kk + 3));
    }
    __device__ __forceinline__ bool vec_ok() const { return true; }
};

// Q (BM points x CC channels x T) for one neighbour slot j = blockIdx.y, contracted over the N outputs in steps of 16.  Thread
// (channel group cg, point group pg) holds PPT points x CPT channels x T.
template <int CPT, int PPT, int CG>
__global__ void __launch_bounds__(256) spider_bwd_data_kernel(const __grid_constant__ SpiderArgs a, const float* __restrict__ W,
                                                              const float* __restrict__ dy, float* __restrict__ D, float* __restrict__ dg) {
    constexpr int T = kTrainT, PG = 256 / CG, BM = PG * PPT, CC = CG * CPT, NCOL = CC * T, BK = 16;
    constexpr int LDY = BM + 4, LDW = NCOL + 4;
    __shared__ __align__(16) float dys[BK][LDY];
    __shared__ __align__(16) float wts[BK][LDW];
    __shared__ float red[CG][BM * T];
    const int tid = threadIdx.x, cg = tid % CG, pg = tid / CG, j = blockIdx.y;
    const long long row0 = (long long)blockIdx.x * BM;
    const int c = a.c, N = a.N, k = a.k;

    float dgacc[PPT][T];
#pragma unroll
    for (int i = 0; i < PPT; ++i)
#pragma unroll
        for (int t = 0; t < T; ++t) dgacc[i][t] = 0.f;

    for (int ch0 = 0; ch0 < c; ch0 += CC) {
        float acc[PPT][CPT * T];
#pragma unroll
        for (int i = 0; i < PPT; ++i)
#pragma unroll
            for (int v = 0; v < CPT * T; ++v) acc[i][v] = 0.f;
        const long long wrow0 = ((long long)j * c + ch0) * T;          // W row of (j, ch0, t = 0)
        const int ncol = min(CC, c - ch0) * T;
        for (int o0 = 0; o0 < N; o0 += BK) {
            __syncthreads();                                           // the previous step's reads are done
            for (int e = tid; e < BM * BK; e += 256) {
                const int pl = e / BK, oo = e - pl * BK;
                const long long p = row0 + pl;
                dys[oo][pl] = (p < a.rows && o0 + oo < N) ? __ldg(dy + p * N + o0 + oo) : 0.f;
            }
            for (int e = tid; e < NCOL * BK; e += 256) {
                const int col = e / BK, oo = e - col * BK;
                wts[oo][col] = (col < ncol && o0 + oo < N) ? __ldg(W + (wrow0 + col) * N + o0 + oo) : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int oo = 0; oo < BK; ++oo) {
                float x[PPT], w[CPT * T];
#pragma unroll
                for (int i = 0; i < PPT; ++i) x[i] = dys[oo][pg * PPT + i];
#pragma unroll
                for (int v = 0; v < CPT * T; ++v) w[v] = wts[oo][cg * CPT * T + v];
#pragma unroll
                for (int i = 0; i < PPT; ++i)
#pragma unroll
                    for (int v = 0; v < CPT * T; ++v) acc[i][v] = fmaf(x[i], w[v], acc[i][v]);
            }
        }
        // epilogue of the chunk: D for these channels, and this thread's channels' share of dg
#pragma unroll
        for (int i = 0; i < PPT; ++i) {
            const long long p = row0 + pg * PPT + i;
            if (p >= a.rows) continue;
            const long long pj = p * k + j;
            float gv[T];
#pragma unroll
            for (int t = 0; t < T; ++t) gv[t] = __ldg(a.g + pj * T + t);
            const int b = (int)(p / a.n);
            const long long nb = (long long)b * a.n + __ldg(a.idx + pj);
#pragma unroll
            for (int u = 0; u < CPT; ++u) {
                const int ch = ch0 + cg * CPT + u;
                if (ch >= c) continue;
                if (D != nullptr) {
                    float s = 0.f;
#pragma unroll
                    for (int t = 0; t < T; ++t) s = fmaf(gv[t], acc[i][u * T + t], s);
                    D[pj * c + ch] = s;
                }
                float h = __ldg(a.feat + nb * c + ch);
                if (a.fs != nullptr) h = fmaxf(fmaf(h, __ldg(a.fs + b * c + ch), __ldg(a.fu + b * c + ch)), 0.f);
#pragma unroll
                for (int t = 0; t < T; ++t) dgacc[i][t] = fmaf(h, acc[i][u * T + t], dgacc[i][t]);
            }
        }
    }
    // dg: the channel groups' shares added in group order
#pragma unroll
    for (int i = 0; i < PPT; ++i)
#pragma unroll
        for (int t = 0; t < T; ++t) red[cg][(pg * PPT + i) * T + t] = dgacc[i][t];
    __syncthreads();
    for (int e = tid; e < BM * T; e += 256) {
        const long long p = row0 + e / T;
        if (p >= a.rows) continue;
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < CG; ++q) s += red[q][e];
        dg[(p * k + j) * T + (e % T)] = s;
    }
}

// d taylor partials: block (T, 64 pair slices); per slice 20 fp64 sums of dg * mono_m over its pairs, folded over the slices in a
// fixed tree -> partial[block][m][t]
constexpr int kTaylorGradBlocks = 4 * kNumSMs;
__global__ void __launch_bounds__(kTrainT * 64) spider_taylor_grad_kernel(long long pairs, const float* __restrict__ delta,
                                                                          const float* __restrict__ dg, double* __restrict__ partial) {
    constexpr int T = kTrainT;
    __shared__ double red[64][T];
    const int t = threadIdx.x, s = threadIdx.y;
    double acc[kTaylorTerms];
#pragma unroll
    for (int m = 0; m < kTaylorTerms; ++m) acc[m] = 0.0;
    for (long long pj = (long long)blockIdx.x * 64 + s; pj < pairs; pj += (long long)gridDim.x * 64) {
        const double X = __ldg(delta + pj * 3), Y = __ldg(delta + pj * 3 + 1), Z = __ldg(delta + pj * 3 + 2);
        const double d = __ldg(dg + pj * T + t);
        // x, y, z, xyz, xy, yz, xz, 1, xx, yy, zz, xxy, xyy, xxz, xzz, yyz, yzz, xxx, yyy, zzz (spider_taylor_kernel's order)
        const double mono[kTaylorTerms] = {X, Y, Z, X * Y * Z, X * Y, Y * Z, X * Z, 1.0, X * X, Y * Y, Z * Z, X * X * Y, X * Y * Y,
                                           X * X * Z, X * Z * Z, Y * Y * Z, Y * Z * Z, X * X * X, Y * Y * Y, Z * Z * Z};
#pragma unroll
        for (int m = 0; m < kTaylorTerms; ++m) acc[m] = fma(d, mono[m], acc[m]);
    }
#pragma unroll
    for (int m = 0; m < kTaylorTerms; ++m) {
        red[s][t] = acc[m];
        __syncthreads();
        for (int w = 32; w > 0; w >>= 1) {
            if (s < w) red[s][t] += red[s + w][t];
            __syncthreads();
        }
        if (s == 0) partial[((size_t)blockIdx.x * kTaylorTerms + m) * T + t] = red[0][t];
        __syncthreads();
    }
}

// dtaylor[m * ld + t] = sum over the blocks' partials, in block order
__global__ void spider_taylor_grad_final_kernel(int nparts, const double* __restrict__ partial, float* __restrict__ dtaylor, int ld) {
    const int e = threadIdx.x;
    if (e >= kTaylorTerms * kTrainT) return;
    double s = 0.0;
    for (int q = 0; q < nparts; ++q) s += partial[(size_t)q * kTaylorTerms * kTrainT + e];
    dtaylor[(e / kTrainT) * ld + e % kTrainT] = (float)s;
}

// Top-2 candidates: (v, i) beats (v', i') when v > v', or v == v' and i < i' (tf.nn.top_k puts the lower index first)
__device__ __forceinline__ void top2_merge(float v, int i, float& v1, int& i1, float& v2, int& i2) {
    if (v > v1 || (v == v1 && i < i1)) { v2 = v1; i2 = i1; v1 = v; i1 = i; }
    else if (v > v2 || (v == v2 && i < i2)) { v2 = v; i2 = i; }
}

// Group norm + ReLU + top-2 pooling backward, block (group, cloud).  Thread (point slice ps, channel cl) visits the same elements
// in the same order as group_norm_affine_kernel, so the fp64 mean and variance are the forward's.  dh of an element = the top-2
// route of dpool + dh_next (the next layer's GroupPointGrad, or null); dz = dh where y * scale + shift > 0.  Writes dy and the
// cloud's dgamma / dbeta partials (b, 2, c) in fp64.
__global__ void __launch_bounds__(256) spider_gn_bwd_kernel(int n, int c, int cpg, float eps, const float* __restrict__ y,
                                                            const float* __restrict__ scale, const float* __restrict__ shift,
                                                            const float* __restrict__ gamma, const float* __restrict__ dpool,
                                                            int pool_channels, int offset, const float* __restrict__ dh_next,
                                                            float* __restrict__ dy, double* __restrict__ partial) {
    __shared__ double red[256];
    __shared__ double cred[2][256];
    __shared__ float tv[2][256];
    __shared__ int ti[2][256];
    const int grp = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int S = 256 / cpg, cl = tid % cpg, ps = tid / cpg, ch = grp * cpg + cl;
    const long long cnt = (long long)n * cpg;
    const float* yb = y + (size_t)b * n * c + ch;
    double s = 0.0;
    for (int p = ps; p < n; p += S) s += (double)__ldg(yb + (size_t)p * c);
    const double mean = block_sum_256(s, red) / (double)cnt;
    double ss = 0.0;
    for (int p = ps; p < n; p += S) {
        const double d = (double)__ldg(yb + (size_t)p * c) - mean;
        ss += d * d;
    }
    const double var = block_sum_256(ss, red) / (double)cnt;
    const double rstd = 1.0 / sqrt(var + (double)eps);

    // the winners of topk_pool_kernel's h = relu(y * scale + shift), per channel
    const float sc = __ldg(scale + (size_t)b * c + ch), sh = __ldg(shift + (size_t)b * c + ch);
    float v1 = -INFINITY, v2 = -INFINITY;
    int i1 = INT_MAX, i2 = INT_MAX;
    for (int p = ps; p < n; p += S) top2_merge(fmaxf(fmaf(__ldg(yb + (size_t)p * c), sc, sh), 0.f), p, v1, i1, v2, i2);
    tv[0][tid] = v1; tv[1][tid] = v2; ti[0][tid] = i1; ti[1][tid] = i2;
    __syncthreads();
    if (ps == 0) {
        for (int q = 1; q < S; ++q) {
            const int o = q * cpg + cl;
            top2_merge(tv[0][o], ti[0][o], v1, i1, v2, i2);
            top2_merge(tv[1][o], ti[1][o], v1, i1, v2, i2);
        }
        ti[0][tid] = i1; ti[1][tid] = i2;
    }
    __syncthreads();
    const int w1 = ti[0][cl], w2 = ti[1][cl];
    const float* dp = dpool + ((size_t)b * pool_channels + offset + ch) * 2;
    const float dp1 = __ldg(dp), dp2 = __ldg(dp + 1);
    const double gm = (double)__ldg(gamma + ch);
    const float* dhb = dh_next != nullptr ? dh_next + (size_t)b * n * c + ch : nullptr;
    auto dz_at = [&](int p, float yv) {
        float d = dhb != nullptr ? __ldg(dhb + (size_t)p * c) : 0.f;
        if (p == w1) d += dp1;
        if (p == w2) d += dp2;
        return fmaf(yv, sc, sh) > 0.f ? d : 0.f;
    };
    double pgam = 0.0, pbet = 0.0;
    for (int p = ps; p < n; p += S) {
        const float yv = __ldg(yb + (size_t)p * c);
        const double dz = (double)dz_at(p, yv), xh = ((double)yv - mean) * rstd;
        pbet += dz;
        pgam += dz * xh;
    }
    const double s1 = block_sum_256(pbet * gm, red);                // sums of gamma * dz and gamma * dz * xhat over the group
    cred[0][tid] = pgam;
    cred[1][tid] = pbet;
    __syncthreads();
    if (ps == 0) {
        double g0 = 0.0, b0 = 0.0;
        for (int q = 0; q < S; ++q) { g0 += cred[0][q * cpg + cl]; b0 += cred[1][q * cpg + cl]; }
        partial[((size_t)b * 2) * c + ch] = g0;
        partial[((size_t)b * 2 + 1) * c + ch] = b0;
    }
    const double s2 = block_sum_256(pgam * gm, red);
    const double m1 = s1 / (double)cnt, m2 = s2 / (double)cnt;
    float* dyb = dy + (size_t)b * n * c + ch;
    for (int p = ps; p < n; p += S) {
        const float yv = __ldg(yb + (size_t)p * c);
        const double xh = ((double)yv - mean) * rstd;
        dyb[(size_t)p * c] = (float)(rstd * (gm * (double)dz_at(p, yv) - m1 - xh * m2));
    }
}

// dgamma[ch], dbeta[ch] = the clouds' partials added in cloud order
__global__ void spider_gn_param_final_kernel(int b, int c, const double* __restrict__ partial, float* __restrict__ dgamma,
                                             float* __restrict__ dbeta) {
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= c) return;
    double g = 0.0, be = 0.0;
    for (int q = 0; q < b; ++q) { g += partial[((size_t)q * 2) * c + ch]; be += partial[((size_t)q * 2 + 1) * c + ch]; }
    dgamma[ch] = (float)g;
    dbeta[ch] = (float)be;
}

static SpiderArgs spider_train_args(int b, int n, int c, int k, int T, int c_out, const int* nn_idx, const float* feat,
                                    const float* fs, const float* fu, const float* g) {
    SpiderArgs a{};
    a.rows = (long long)b * n; a.n = n; a.c = c; a.k = k; a.T = T; a.K = k * T * c; a.N = c_out;
    a.feat = feat; a.idx = nn_idx; a.g = g; a.fs = fs; a.fu = fu;
    return a;
}

static int spider_weight_splits(long long rows, long long K, int N, long long* kps) {
    return weight_grad_splits(rows, (int)(((K + 127) / 128) * ((N + 63) / 64)), kps);
}

}  // namespace psa

using namespace psa;

extern "C" size_t psa_spider_conv_workspace_bytes(int b, int n, int c, int k, int T, int c_out) {
    if (b < 0 || n < 1 || c < 1 || k < 1 || k > kSpiderMaxK || T < 1 || c_out < 1) return 0;
    return spider_ws(b, n, c, k, T, c_out).total;
}

extern "C" int psa_spider_conv_infer(int b, int n, int c, int k, int T, int c_out, const float* delta, const int* nn_idx,
                                     const float* feat, const float* feat_scale, const float* feat_shift, const float* taylor,
                                     const float* W, const float* bias, float* y, void* workspace, size_t workspace_bytes,
                                     psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 1 && c >= 1 && T >= 1 && c_out >= 1, "spider_conv: bad dims b=%d n=%d c=%d T=%d c_out=%d", b, n, c, T, c_out);
    PSA_REQUIRE(k >= 1 && k <= kSpiderMaxK, "spider_conv: k=%d must be in [1, %d]", k, kSpiderMaxK);
    PSA_REQUIRE((long long)k * T * c <= (1LL << 30), "spider_conv: k*T*c too large");
    PSA_REQUIRE((feat_scale == nullptr) == (feat_shift == nullptr), "spider_conv: feat_scale and feat_shift are given together or not at all");
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(delta && nn_idx && feat && taylor && W && bias && y, "spider_conv: null buffer");
    const SpiderWs ws = spider_ws(b, n, c, k, T, c_out);
    PSA_REQUIRE(workspace != nullptr && workspace_bytes >= ws.total,
                "spider_conv: workspace of %zu bytes required (psa_spider_conv_workspace_bytes), got %zu", ws.total, workspace_bytes);
    PSA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "spider_conv: workspace must be 256-byte aligned");
    cudaStream_t st = as_stream(stream);
    uint8_t* wsb = reinterpret_cast<uint8_t*>(workspace);
    const long long rows = (long long)b * n, pairs = rows * k;
    SpiderArgs a;
    a.rows = rows; a.n = n; a.c = c; a.k = k; a.T = T; a.K = k * T * c; a.N = c_out;
    a.feat = feat; a.idx = nn_idx; a.g = reinterpret_cast<float*>(wsb + ws.g); a.fs = feat_scale; a.fu = feat_shift;
    a.bias = bias; a.y = y;
    spider_taylor_kernel<<<(unsigned)((pairs * T + 255) / 256), 256, 0, st>>>(pairs, T, delta, taylor, const_cast<float*>(a.g));
    int rc = check_launch("spider_taylor_kernel");
    if (rc != PSA_OK) return rc;
    if (mlp_mode() == 1 || !spider_tc_eligible(rows, c, k, T, c_out, feat, feat_scale, feat_shift, bias, y)) {
        const dim3 grid((unsigned)((rows + 63) / 64), (unsigned)((c_out + 63) / 64));
        spider_fma_kernel<<<grid, 256, 0, st>>>(a, W);
        return check_launch("spider_fma_kernel");
    }
    const int K = a.K, Nt = tc_dense_nt(rows, c_out) & ~kImageFlags;
    float* wp = reinterpret_cast<float*>(wsb + ws.wp);
    spider_permute_kernel<<<1024, 256, 0, st>>>(k, c, T, c_out, W, wp);
    rc = check_launch("spider_permute_kernel");
    if (rc != PSA_OK) return rc;
    PSA_CUDA(cudaMemsetAsync(wsb, 0, 256, st));
    return ring_run(kSpiderRing, a, (rows + 127) / 128 * (c_out / Nt), RingWeights{K, K, c_out, Nt, wp, wsb + ws.img2, wsb + ws.img3},
                    reinterpret_cast<unsigned int*>(wsb), nullptr, st);
}

extern "C" int psa_group_norm_affine(int b, int n, int c, int groups, float eps, const float* y, const float* gamma,
                                     const float* beta, float* scale, float* shift, float* out, int relu, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 1 && c >= 1 && groups >= 1, "group_norm_affine: bad dims b=%d n=%d c=%d groups=%d", b, n, c, groups);
    PSA_REQUIRE(c % groups == 0, "group_norm_affine: %d groups do not divide %d channels", groups, c);
    PSA_REQUIRE(eps >= 0.f, "group_norm_affine: eps must be >= 0");
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(y && gamma && beta && scale && shift, "group_norm_affine: null buffer");
    cudaStream_t st = as_stream(stream);
    group_norm_affine_kernel<<<dim3((unsigned)groups, (unsigned)b), 256, 0, st>>>(n, c, c / groups, eps, y, gamma, beta, scale, shift);
    int rc = check_launch("group_norm_affine_kernel");
    if (rc != PSA_OK || out == nullptr) return rc;
    const long long total = (long long)b * n * c;
    cloud_affine_kernel<<<(unsigned)min((total + 255) / 256, 8192LL), 256, 0, st>>>(total, n, c, y, scale, shift, relu, out);
    return check_launch("cloud_affine_kernel");
}

extern "C" int psa_topk_pool(int b, int n, int c, int k, const float* y, const float* scale, const float* shift, int relu,
                             float* out, int out_channels, int offset, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && c >= 1 && offset >= 0 && offset + c <= out_channels, "topk_pool: bad dims b=%d c=%d offset=%d out_channels=%d",
                b, c, offset, out_channels);
    PSA_SUPPORTED(k == 2, "topk_pool: only k = 2 (SpiderCNN's pooling) is compiled in, got k=%d", k);
    PSA_REQUIRE(n >= k, "topk_pool: n=%d points, fewer than k=%d", n, k);
    PSA_REQUIRE((scale == nullptr) == (shift == nullptr), "topk_pool: scale and shift are given together or not at all");
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(y && out, "topk_pool: null buffer");
    topk_pool_kernel<<<dim3((unsigned)((c + 31) / 32), (unsigned)b), dim3(32, 8), 0, as_stream(stream)>>>(n, c, y, scale, shift, relu, out,
                                                                                                        out_channels, offset);
    return check_launch("topk_pool_kernel");
}

extern "C" int psa_spider_taylor_filter(int b, int n, int k, int T, const float* delta, const float* taylor, float* g, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 1 && k >= 1 && T >= 1, "spider_taylor_filter: bad dims b=%d n=%d k=%d T=%d", b, n, k, T);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(delta && taylor && g, "spider_taylor_filter: null buffer");
    const long long pairs = (long long)b * n * k;
    spider_taylor_kernel<<<(unsigned)((pairs * T + 255) / 256), 256, 0, as_stream(stream)>>>(pairs, T, delta, taylor, g);
    return check_launch("spider_taylor_kernel");
}

static int spider_bwd_dims(const char* what, int b, int n, int c, int k, int T, int c_out) {
    PSA_REQUIRE(b >= 0 && n >= 1 && c >= 1 && c_out >= 1, "%s: bad dims b=%d n=%d c=%d c_out=%d", what, b, n, c, c_out);
    PSA_REQUIRE(k >= 1 && k <= kSpiderMaxK, "%s: k=%d must be in [1, %d]", what, k, kSpiderMaxK);
    PSA_REQUIRE((long long)k * T * c <= (1LL << 30), "%s: k*T*c too large", what);
    PSA_SUPPORTED(T == kTrainT, "%s: only T = %d (SpiderCNN's taylor_channel) is compiled in, got T=%d", what, kTrainT, T);
    return PSA_OK;
}

extern "C" size_t psa_spider_conv_bwd_workspace_bytes(int b, int n, int c, int k, int T, int c_out) {
    if (b < 0 || n < 1 || c < 1 || k < 1 || k > kSpiderMaxK || T != kTrainT || c_out < 1) return 0;
    long long kps;
    const long long K = (long long)k * T * c;
    const int splits = spider_weight_splits((long long)b * n, K, c_out, &kps);
    size_t bytes = splits > 1 ? (size_t)splits * K * c_out * sizeof(float) : 0;
    bytes = max(bytes, (size_t)kTaylorGradBlocks * kTaylorTerms * kTrainT * sizeof(double));
    bytes = max(bytes, (size_t)b * 2 * c * sizeof(double));
    return al256(bytes);
}

extern "C" int psa_spider_conv_bwd_weight(int b, int n, int c, int k, int T, int c_out, const int* nn_idx, const float* feat,
                                          const float* feat_scale, const float* feat_shift, const float* g, const float* dy, float* dW,
                                          void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = spider_bwd_dims("spider_conv_bwd_weight", b, n, c, k, T, c_out);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE((feat_scale == nullptr) == (feat_shift == nullptr), "spider_conv_bwd_weight: feat_scale and feat_shift are given together or not at all");
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(nn_idx && feat && g && dy && dW, "spider_conv_bwd_weight: null buffer");
    cudaStream_t st = as_stream(stream);
    const long long rows = (long long)b * n, K = (long long)k * T * c;
    long long kps;
    const int splits = spider_weight_splits(rows, K, c_out, &kps);
    GemmOut o;
    o.ld_out = c_out; o.bias = nullptr; o.col_skip = 0; o.stat_partial = nullptr;
    o.out = dW;
    if (splits > 1) {
        PSA_REQUIRE(workspace != nullptr && workspace_bytes >= (size_t)splits * K * c_out * sizeof(float),
                    "spider_conv_bwd_weight: workspace too small (psa_spider_conv_bwd_workspace_bytes)");
        o.out = reinterpret_cast<float*>(workspace);
    }
    const SpiderA fa{spider_train_args(b, n, c, k, T, c_out, nn_idx, feat, feat_scale, feat_shift, g)};
    const MatIn fb{dy, c_out};
    // 128 x 64 tiles only: the gathered operand's index arithmetic does not fit 128 x 128's two CTAs per SM without spills
    const dim3 grid((unsigned)((c_out + 63) / 64), (unsigned)((K + 127) / 128), (unsigned)splits);
    train_gemm_kernel<128, 64, false, true><<<grid, kGemmThreads, 0, st>>>(fa, fb, o, K, c_out, rows, kps);
    rc = check_launch("train_gemm_kernel");
    if (rc != PSA_OK || splits == 1) return rc;
    return reduce_partials(splits, (int)(K * c_out), o.out, dW, st);
}

extern "C" int psa_spider_conv_bwd_data(int b, int n, int c, int k, int T, int c_out, const int* nn_idx, const float* feat,
                                        const float* feat_scale, const float* feat_shift, const float* g, const float* W, const float* dy,
                                        float* D, float* dg, psa_stream_t stream) {
    int rc = spider_bwd_dims("spider_conv_bwd_data", b, n, c, k, T, c_out);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE((feat_scale == nullptr) == (feat_shift == nullptr), "spider_conv_bwd_data: feat_scale and feat_shift are given together or not at all");
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(nn_idx && feat && g && W && dy && dg, "spider_conv_bwd_data: null buffer");
    const SpiderArgs a = spider_train_args(b, n, c, k, T, c_out, nn_idx, feat, feat_scale, feat_shift, g);
    cudaStream_t st = as_stream(stream);
    if (c % 32 == 0)       // 64 points x 32 channels per chunk
        spider_bwd_data_kernel<2, 4, 16><<<dim3((unsigned)((a.rows + 63) / 64), (unsigned)k), 256, 0, st>>>(a, W, dy, D, dg);
    else                   // 128 points x 4 channels per chunk (the first layer's c = 3)
        spider_bwd_data_kernel<1, 2, 4><<<dim3((unsigned)((a.rows + 127) / 128), (unsigned)k), 256, 0, st>>>(a, W, dy, D, dg);
    return check_launch("spider_bwd_data_kernel");
}

extern "C" int psa_spider_taylor_grad(int b, int n, int k, int T, const float* delta, const float* dg, float* dtaylor, int ld_taylor,
                                      void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 1 && k >= 1, "spider_taylor_grad: bad dims b=%d n=%d k=%d", b, n, k);
    PSA_SUPPORTED(T == kTrainT, "spider_taylor_grad: only T = %d is compiled in, got T=%d", kTrainT, T);
    PSA_REQUIRE(ld_taylor >= T, "spider_taylor_grad: ld_taylor=%d < T=%d", ld_taylor, T);
    PSA_REQUIRE(dtaylor != nullptr, "spider_taylor_grad: null buffer");
    cudaStream_t st = as_stream(stream);
    const long long pairs = (long long)b * n * k;
    const int blocks = (int)min((long long)kTaylorGradBlocks, max(1LL, (pairs + 63) / 64));
    PSA_REQUIRE(pairs == 0 || (delta && dg), "spider_taylor_grad: null buffer");
    PSA_REQUIRE(workspace != nullptr && workspace_bytes >= (size_t)blocks * kTaylorTerms * kTrainT * sizeof(double),
                "spider_taylor_grad: workspace too small (psa_spider_conv_bwd_workspace_bytes)");
    double* partial = reinterpret_cast<double*>(workspace);
    spider_taylor_grad_kernel<<<blocks, dim3(kTrainT, 64), 0, st>>>(pairs, delta, dg, partial);
    int rc = check_launch("spider_taylor_grad_kernel");
    if (rc != PSA_OK) return rc;
    spider_taylor_grad_final_kernel<<<1, 128, 0, st>>>(blocks, partial, dtaylor, ld_taylor);
    return check_launch("spider_taylor_grad_final_kernel");
}

extern "C" int psa_spider_gn_bwd(int b, int n, int c, int groups, float eps, const float* y, const float* scale, const float* shift,
                                 const float* gamma, const float* dpool, int pool_channels, int offset, const float* dh_next, float* dy,
                                 float* dgamma, float* dbeta, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 2 && c >= 1 && groups >= 1, "spider_gn_bwd: bad dims b=%d n=%d c=%d groups=%d", b, n, c, groups);
    PSA_REQUIRE(c % groups == 0, "spider_gn_bwd: %d groups do not divide %d channels", groups, c);
    PSA_SUPPORTED(256 % (c / groups) == 0, "spider_gn_bwd: %d channels per group must divide 256", c / groups);
    PSA_REQUIRE(eps >= 0.f, "spider_gn_bwd: eps must be >= 0");
    PSA_REQUIRE(offset >= 0 && offset + c <= pool_channels, "spider_gn_bwd: offset=%d + c=%d exceeds pool_channels=%d", offset, c, pool_channels);
    PSA_REQUIRE(dgamma && dbeta, "spider_gn_bwd: null buffer");
    cudaStream_t st = as_stream(stream);
    PSA_REQUIRE(workspace != nullptr && workspace_bytes >= (size_t)b * 2 * c * sizeof(double),
                "spider_gn_bwd: workspace too small (psa_spider_conv_bwd_workspace_bytes)");
    double* partial = reinterpret_cast<double*>(workspace);
    if (b > 0) {
        PSA_REQUIRE(y && scale && shift && gamma && dpool && dy, "spider_gn_bwd: null buffer");
        spider_gn_bwd_kernel<<<dim3((unsigned)groups, (unsigned)b), 256, 0, st>>>(n, c, c / groups, eps, y, scale, shift, gamma, dpool,
                                                                               pool_channels, offset, dh_next, dy, partial);
        int rc = check_launch("spider_gn_bwd_kernel");
        if (rc != PSA_OK) return rc;
    }
    spider_gn_param_final_kernel<<<(c + 127) / 128, 128, 0, st>>>(b, c, partial, dgamma, dbeta);
    return check_launch("spider_gn_param_final_kernel");
}
