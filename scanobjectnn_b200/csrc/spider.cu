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
#include <float.h>

#include "common.cuh"
#include "ring_gemm.cuh"

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
