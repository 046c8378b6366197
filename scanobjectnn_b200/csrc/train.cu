// train.cu -- training mode of the point-set-abstraction path: batch-statistics BN, max-pool with arg routing, the
// backward pass of a level and of the FC head, loss, Adam.  See include/psa.h ("Training mode") for the contract and
// train_gemm.cuh for the fused GEMM all the dense products run on.
//
// Determinism: every reduction here (column statistics, BN backward sums, split-K weight gradients, the GroupPointGrad
// scatter) is a fixed-order sum -- per-CTA partials in a fixed thread order, partials added in index order in fp64.  The
// reference's gradient kernels are float atomicAdd scatters (tf_grouping_g.cu:61-78, tf_sampling_g.cu:183-192).
#include <math.h>

#include "train_gemm.cuh"

namespace psa {

// tensor-core forward of a training layer (tc_mlp.cu): operands split into three bf16 pieces, fp32 accumulation
bool tc_train_fwd_eligible(long long rows, int K, int N);
size_t tc_dense_image_bytes(int K, int N);
int launch_tc_dense_train(long long rows, int K, int N, const float* x, const float* in_scale, const float* in_shift, int in_relu,
                          const float* W, const float* bias, float* y, float* stat_partial, uint8_t* image_ws, cudaStream_t st);

// out[e] = sum_p partial[p * len + e] in a FIXED tree: block = 32 outputs x 32 chunk lanes; lane c adds its contiguous range of
// partials in ascending order (fp64, eight loads in flight), the 32 chunk sums are added in lane order.  Deterministic, and
// ~32x shorter dependent chains than one thread per output (4096 tile partials took 290 us that way).
__global__ void __launch_bounds__(1024) reduce_partials_kernel(int nparts, int len, const float* __restrict__ partial, float* __restrict__ out) {
    __shared__ double red[32][33];
    const int ex = threadIdx.x & 31, cl = threadIdx.x >> 5;
    const int e = blockIdx.x * 32 + ex;
    const int per = (nparts + 31) / 32;
    const int p0 = cl * per, p1 = min(nparts, p0 + per);
    double s = 0.0;
    if (e < len) {
        int p = p0;
        for (; p + 7 < p1; p += 8) {
            float v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = __ldcg(partial + (size_t)(p + u) * len + e);
#pragma unroll
            for (int u = 0; u < 8; ++u) s += (double)v[u];
        }
        for (; p < p1; ++p) s += (double)__ldcg(partial + (size_t)p * len + e);
    }
    red[cl][ex] = s;
    __syncthreads();
    if (cl == 0 && e < len) {
        double t = 0.0;
#pragma unroll
        for (int c = 0; c < 32; ++c) t += red[c][ex];
        out[e] = (float)t;
    }
}

int reduce_partials(int nparts, int len, const float* partial, float* out, cudaStream_t st) {
    reduce_partials_kernel<<<(len + 31) / 32, 1024, 0, st>>>(nparts, len, partial, out);
    return check_launch("reduce_partials_kernel");
}

template <int BM, int BN, bool A_KC, bool B_NC, bool GROUP = false, class FA, class FB>
static int launch_gemm(const FA& fa, const FB& fb, const GemmOut& o, long long M, int N, long long Kc, int splits, long long k_per_split,
                       cudaStream_t st) {
    dim3 grid((unsigned)((N + BN - 1) / BN), (unsigned)((M + BM - 1) / BM), (unsigned)splits);
    train_gemm_kernel<BM, BN, A_KC, B_NC, FA, FB, GROUP><<<grid, kGemmThreads, 0, st>>>(fa, fb, o, M, N, Kc, k_per_split);
    return check_launch("train_gemm_kernel");
}

// ---- small-M products (the FC head: rows = batch): contraction split over CTAs, finished here in split order ----
// out[m][n - col_skip] = sum_z partial[z][m][n] (+ bias[n]);  grid over M*N elements
__global__ void splitk_finish_kernel(int splits, long long M, int N, const float* __restrict__ partial, const float* __restrict__ bias,
                                     float* __restrict__ out, long long ld_out, int col_skip) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= M * N) return;
    const long long m = e / N;
    const int n = (int)(e - m * N);
    float t = 0.f;
    for (int z = 0; z < splits; ++z) t += partial[(size_t)z * M * N + e];
    if (bias != nullptr) t += __ldg(bias + n);
    if (n >= col_skip) out[m * ld_out + (n - col_skip)] = t;
}
// stats (2, N) of y (M, N), M small: block = 32 columns x 32 row lanes, fixed-order tree
__global__ void __launch_bounds__(1024) col_stats_kernel(long long M, int N, const float* __restrict__ y, float* __restrict__ stats) {
    __shared__ double red[2][32][33];
    const int ex = threadIdx.x & 31, rl = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + ex;
    double s = 0.0, q = 0.0;
    if (n < N)
        for (long long m = rl; m < M; m += 32) { const double v = y[m * N + n]; s += v; q += v * v; }
    red[0][rl][ex] = s; red[1][rl][ex] = q;
    __syncthreads();
    if (rl == 0 && n < N) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int k = 0; k < 32; ++k) { a += red[0][k][ex]; b += red[1][k][ex]; }
        stats[n] = (float)a; stats[N + n] = (float)b;
    }
}

// ---- batch-norm finalize ----
// one channel: batch mean and biased variance -> scale / shift, mean_inv, moving averages
__device__ __forceinline__ void bn_finalize_channel(int C, int c, double mean, double var, const float* __restrict__ gamma,
                                                    const float* __restrict__ beta, float decay, float* __restrict__ moving_mean,
                                                    float* __restrict__ moving_var, float* __restrict__ scale, float* __restrict__ shift,
                                                    float* __restrict__ mean_inv) {
    if (var < 0.0) var = 0.0;
    const double inv = 1.0 / sqrt(var + 1e-3);
    const float sc = (float)((double)gamma[c] * inv);
    scale[c] = sc;
    shift[c] = (float)((double)beta[c] - mean * (double)gamma[c] * inv);
    if (mean_inv != nullptr) { mean_inv[c] = (float)mean; mean_inv[C + c] = (float)inv; }
    if (moving_mean != nullptr) moving_mean[c] = decay * moving_mean[c] + (1.f - decay) * (float)mean;
    if (moving_var != nullptr) moving_var[c] = decay * moving_var[c] + (1.f - decay) * (float)var;
}

__global__ void bn_finalize_kernel(int C, double inv_count, const float* __restrict__ stats, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float decay, float* __restrict__ moving_mean,
                                   float* __restrict__ moving_var, float* __restrict__ scale, float* __restrict__ shift,
                                   float* __restrict__ mean_inv) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const double mean = (double)stats[c] * inv_count;
    const double var = (double)stats[C + c] * inv_count - mean * mean;    // biased (tf.nn.moments / contrib batch_norm)
    bn_finalize_channel(C, c, mean, var, gamma, beta, decay, moving_mean, moving_var, scale, shift, mean_inv);
}

// the same from a materialised y (M, N) in two fp64 passes: the mean, then the centred sum of squares.  E[y^2] - mean^2 from fp32
// sums loses the variance of a column whose mean is large against its spread: DGCNN's fc1 / T-net tfc1 after the max over the
// points, where mean^2 / var reaches ~4000 and 1/sigma lost ~1e-4.  Block = 32 columns x 32 row lanes, fixed-order tree.
__global__ void __launch_bounds__(1024)
bn_finalize_rows_kernel(long long M, int N, const float* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                        float decay, float* __restrict__ moving_mean, float* __restrict__ moving_var, float* __restrict__ scale,
                        float* __restrict__ shift, float* __restrict__ mean_inv) {
    __shared__ double red[32][33];
    __shared__ double mean_s[32];
    const int ex = threadIdx.x & 31, rl = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + ex;
    double s = 0.0;
    if (n < N)
        for (long long m = rl; m < M; m += 32) s += (double)y[m * N + n];
    red[rl][ex] = s;
    __syncthreads();
    if (rl == 0) {
        double a = 0.0;
#pragma unroll
        for (int k = 0; k < 32; ++k) a += red[k][ex];
        mean_s[ex] = a / (double)M;
    }
    __syncthreads();
    const double mean = mean_s[ex];
    double q = 0.0;
    if (n < N)
        for (long long m = rl; m < M; m += 32) { const double d = (double)y[m * N + n] - mean; q += d * d; }
    red[rl][ex] = q;                                           // the mean's tree was read before the barrier above
    __syncthreads();
    if (rl == 0 && n < N) {
        double b = 0.0;
#pragma unroll
        for (int k = 0; k < 32; ++k) b += red[k][ex];
        bn_finalize_channel(N, n, mean, b / (double)M, gamma, beta, decay, moving_mean, moving_var, scale, shift, mean_inv);
    }
}

// ---- max-pool over runs of pool_k rows with the first winning row ----
__global__ void train_pool_fwd_kernel(long long groups, int pool_k, int C4, const float4* __restrict__ y, const float4* __restrict__ scale,
                                      const float4* __restrict__ shift, float4* __restrict__ pooled, int4* __restrict__ argk) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= groups * C4) return;
    const long long g = e / C4;
    const int c4 = (int)(e - g * C4);
    const float4 s = __ldg(scale + c4), t = __ldg(shift + c4);
    float4 best = make_float4(-1.f, -1.f, -1.f, -1.f);                 // relu output is >= 0: row 0 always beats the sentinel
    int4 arg = make_int4(0, 0, 0, 0);
    const float4* row = y + (size_t)g * pool_k * C4 + c4;
    for (int k = 0; k < pool_k; ++k) {
        const float4 v = __ldg(row + (size_t)k * C4);
        const float zx = fmaxf(fmaf(v.x, s.x, t.x), 0.f), zy = fmaxf(fmaf(v.y, s.y, t.y), 0.f);
        const float zz = fmaxf(fmaf(v.z, s.z, t.z), 0.f), zw = fmaxf(fmaf(v.w, s.w, t.w), 0.f);
        if (zx > best.x) { best.x = zx; arg.x = k; }
        if (zy > best.y) { best.y = zy; arg.y = k; }
        if (zz > best.z) { best.z = zz; arg.z = k; }
        if (zw > best.w) { best.w = zw; arg.w = k; }
    }
    pooled[e] = best;
    argk[e] = arg;
}

// ---- pooling over runs of pool_k rows, the modes of pointnet_util.py:126-146 other than the fused max ----
// mode 0: max, 1: avg (reduce_mean), 2: weighted_avg with w_k = exp(-5 d_k) / sum_k exp(-5 d_k), d = |grouped_xyz| per row
__global__ void pool_rows_kernel(long long groups, int pool_k, int C4, int mode, const float4* __restrict__ x, const float* __restrict__ dist,
                                 float4* __restrict__ out) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= groups * C4) return;
    const long long g = e / C4;
    const int c4 = (int)(e - g * C4);
    const float4* row = x + (size_t)g * pool_k * C4 + c4;
    float4 acc;
    if (mode == 0) {
        acc = __ldg(row);
        for (int k = 1; k < pool_k; ++k) {
            const float4 v = __ldg(row + (size_t)k * C4);
            acc.x = fmaxf(acc.x, v.x); acc.y = fmaxf(acc.y, v.y); acc.z = fmaxf(acc.z, v.z); acc.w = fmaxf(acc.w, v.w);
        }
    } else {
        acc = make_float4(0.f, 0.f, 0.f, 0.f);
        float wsum = 0.f;
        for (int k = 0; k < pool_k; ++k) {
            const float4 v = __ldg(row + (size_t)k * C4);
            const float w = mode == 2 ? expf(-5.f * __ldg(dist + (size_t)g * pool_k + k)) : 1.f;
            wsum += w;
            acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
        }
        const float inv = 1.f / wsum;
        acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
    }
    out[e] = acc;
}

// ---- batch-norm backward sums ----
// block = (C/4 channel quads) x RL row lanes; each block owns a contiguous chunk of rows; partial (blocks, 2, C)
constexpr int kBnbThreads = 256;

__global__ void __launch_bounds__(kBnbThreads)
bn_bwd_partial_kernel(const GradIn g, long long rows, int C, const float* __restrict__ mean_inv, long long rows_per_block,
                      float* __restrict__ partial) {
    __shared__ float red[kBnbThreads * 8];
    const int C4 = C / 4;
    const int RL = kBnbThreads / C4;                                  // row lanes (>= 1 for C <= 1024)
    const int cq = threadIdx.x % C4, rl = threadIdx.x / C4;
    float4 sb = make_float4(0.f, 0.f, 0.f, 0.f), sg = sb;
    if (rl < RL) {
        const int c = cq * 4;
        const float4 mu = __ldg(reinterpret_cast<const float4*>(mean_inv + c)), inv = __ldg(reinterpret_cast<const float4*>(mean_inv + C + c));
        const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
        if (g.mode == 0) {
            for (long long r = r0 + rl; r < r1; r += RL) {
                // y itself, not g.y4: that reads zeros without a relu gate (s == NULL), and xhat needs y in every case
                const float4 yv = __ldg(reinterpret_cast<const float4*>(g.y + r * g.ld + c));
                const float4 dz = g.dz4(r, c, yv);
                sb.x += dz.x; sb.y += dz.y; sb.z += dz.z; sb.w += dz.w;
                sg.x = fmaf(dz.x, (yv.x - mu.x) * inv.x, sg.x); sg.y = fmaf(dz.y, (yv.y - mu.y) * inv.y, sg.y);
                sg.z = fmaf(dz.z, (yv.z - mu.z) * inv.z, sg.z); sg.w = fmaf(dz.w, (yv.w - mu.w) * inv.w, sg.w);
            }
        } else {
            // pooled routing: `rows` counts GROUPS here; only the winning row of each (group, channel) carries gradient
            for (long long gi = r0 + rl; gi < r1; gi += RL) {
                const size_t o = (size_t)gi * C + c;
                const int4 a = __ldg(reinterpret_cast<const int4*>(g.argk + o));
                const float4 p = __ldg(reinterpret_cast<const float4*>(g.pv + o)), d = __ldg(reinterpret_cast<const float4*>(g.dp + o));
                const float* yb = g.y + (size_t)gi * g.pool_k * g.ld + c;
                if (p.x > 0.f) { const float yv = __ldg(yb + (size_t)a.x * g.ld + 0); sb.x += d.x; sg.x = fmaf(d.x, (yv - mu.x) * inv.x, sg.x); }
                if (p.y > 0.f) { const float yv = __ldg(yb + (size_t)a.y * g.ld + 1); sb.y += d.y; sg.y = fmaf(d.y, (yv - mu.y) * inv.y, sg.y); }
                if (p.z > 0.f) { const float yv = __ldg(yb + (size_t)a.z * g.ld + 2); sb.z += d.z; sg.z = fmaf(d.z, (yv - mu.z) * inv.z, sg.z); }
                if (p.w > 0.f) { const float yv = __ldg(yb + (size_t)a.w * g.ld + 3); sb.w += d.w; sg.w = fmaf(d.w, (yv - mu.w) * inv.w, sg.w); }
            }
        }
    }
    float* mine = red + threadIdx.x * 8;
    mine[0] = sb.x; mine[1] = sb.y; mine[2] = sb.z; mine[3] = sb.w; mine[4] = sg.x; mine[5] = sg.y; mine[6] = sg.z; mine[7] = sg.w;
    __syncthreads();
    float* dst = partial + (size_t)blockIdx.x * 2 * C;
    for (int e = threadIdx.x; e < 2 * C; e += kBnbThreads) {
        const int which = e / C, c = e - which * C;
        float t = 0.f;
        for (int r = 0; r < RL; ++r) t += red[(r * C4 + (c >> 2)) * 8 + which * 4 + (c & 3)];      // row lanes in order
        dst[e] = t;
    }
}

__global__ void __launch_bounds__(1024)
bn_bwd_final_kernel(int nparts, int C, double inv_rows, const float* __restrict__ partial, const float* __restrict__ gamma,
                    const float* __restrict__ mean_inv, float* __restrict__ dgamma, float* __restrict__ dbeta,
                    float* __restrict__ ca, float* __restrict__ cb, float* __restrict__ cc) {
    __shared__ double red[2][32][33];
    const int ex = threadIdx.x & 31, cl = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + ex;
    const int per = (nparts + 31) / 32;
    const int p0 = cl * per, p1 = min(nparts, p0 + per);
    double sb = 0.0, sg = 0.0;
    if (c < C) {
        int p = p0;
        for (; p + 3 < p1; p += 4) {
            float vb[4], vg[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) { vb[u] = __ldcg(partial + (size_t)(p + u) * 2 * C + c); vg[u] = __ldcg(partial + (size_t)(p + u) * 2 * C + C + c); }
#pragma unroll
            for (int u = 0; u < 4; ++u) { sb += (double)vb[u]; sg += (double)vg[u]; }
        }
        for (; p < p1; ++p) { sb += (double)__ldcg(partial + (size_t)p * 2 * C + c); sg += (double)__ldcg(partial + (size_t)p * 2 * C + C + c); }
    }
    red[0][cl][ex] = sb;
    red[1][cl][ex] = sg;
    __syncthreads();
    if (cl != 0 || c >= C) return;
    double db = 0.0, dg = 0.0;
#pragma unroll
    for (int k = 0; k < 32; ++k) { db += red[0][k][ex]; dg += red[1][k][ex]; }
    dbeta[c] = (float)db;
    dgamma[c] = (float)dg;
    const double gm = gamma[c], mu = mean_inv[c], inv = mean_inv[C + c];
    // dy = gamma*inv/R * (R dz - dbeta - xhat dgamma),  xhat = (y - mu) inv
    ca[c] = (float)(gm * inv);
    cb[c] = (float)(-gm * inv * inv * dg * inv_rows);
    cc[c] = (float)(gm * inv * (mu * inv * dg - db) * inv_rows);
}

int launch_bn_bwd_final(int nparts, int C, long long rows, const float* partial, const float* gamma, const float* mean_inv, float* dgamma,
                        float* dbeta, float* ca, float* cb, float* cc, cudaStream_t st) {
    bn_bwd_final_kernel<<<(C + 31) / 32, 1024, 0, st>>>(nparts, C, 1.0 / (double)rows, partial, gamma, mean_inv, dgamma, dbeta, ca, cb, cc);
    return check_launch("bn_bwd_final_kernel");
}

// ---- first-layer backward of a set-abstraction level ----
// dW_xyz partials: block = (C1/4 quads) x row lanes over a contiguous chunk of grouped rows
__global__ void __launch_bounds__(kBnbThreads)
conv1_dwxyz_partial_kernel(const GradIn g, long long rows, int nsample, long long rows_per_cloud, int n, int m, int C1,
                           const float* __restrict__ xyz, const float* __restrict__ new_xyz, const int* __restrict__ idx,
                           long long rows_per_block, float* __restrict__ partial) {
    __shared__ float red[kBnbThreads * 12];
    const int C4 = C1 / 4, RL = kBnbThreads / C4;
    const int cq = threadIdx.x % C4, rl = threadIdx.x / C4;
    float acc[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) acc[i] = 0.f;
    if (rl < RL) {
        const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
        for (long long r = r0 + rl; r < r1; r += RL) {
            const long long cloud = r / rows_per_cloud;
            const long long q = r / nsample;                               // global query id
            const int j = __ldg(idx + r);
            const float* p = xyz + ((size_t)cloud * n + j) * 3;
            const float* cq3 = new_xyz + (size_t)q * 3;
            const float dx = __ldg(p) - __ldg(cq3), dy = __ldg(p + 1) - __ldg(cq3 + 1), dz = __ldg(p + 2) - __ldg(cq3 + 2);
            const float4 gy = g.get4(r, cq * 4);
            acc[0] = fmaf(dx, gy.x, acc[0]); acc[1] = fmaf(dx, gy.y, acc[1]); acc[2] = fmaf(dx, gy.z, acc[2]); acc[3] = fmaf(dx, gy.w, acc[3]);
            acc[4] = fmaf(dy, gy.x, acc[4]); acc[5] = fmaf(dy, gy.y, acc[5]); acc[6] = fmaf(dy, gy.z, acc[6]); acc[7] = fmaf(dy, gy.w, acc[7]);
            acc[8] = fmaf(dz, gy.x, acc[8]); acc[9] = fmaf(dz, gy.y, acc[9]); acc[10] = fmaf(dz, gy.z, acc[10]); acc[11] = fmaf(dz, gy.w, acc[11]);
        }
    }
    (void)m;
#pragma unroll
    for (int i = 0; i < 12; ++i) red[threadIdx.x * 12 + i] = acc[i];
    __syncthreads();
    float* dst = partial + (size_t)blockIdx.x * 3 * C1;
    for (int e = threadIdx.x; e < 3 * C1; e += kBnbThreads) {
        const int ax = e / C1, c = e - ax * C1;
        float t = 0.f;
        for (int r = 0; r < RL; ++r) t += red[(r * C4 + (c >> 2)) * 12 + ax * 4 + (c & 3)];
        dst[e] = t;
    }
}

// GroupPointGrad of the training path: CSR built by scatter.cu's stable counting sort (launch_group_csr), then one warp per
// source point (lane = 4 channels) adds the rows of the point in list order.  Fixed order => bit-reproducible.
__global__ void __launch_bounds__(256)
group_grad_csr_kernel(const GradIn g, int n, int mk, int C1, long long total_points, const int* __restrict__ offsets, const int* __restrict__ list,
                      float* __restrict__ dU) {
    const int lane = threadIdx.x & 31;
    const long long pt = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);           // global source point b*n + j
    if (pt >= total_points) return;
    const long long cloud = pt / n;
    const int j = (int)(pt - cloud * n);
    const int* off = offsets + (size_t)cloud * (n + 1);
    const int* lst = list + (size_t)cloud * mk;
    const int t0 = __ldg(off + j), t1 = __ldg(off + j + 1);
    for (int c0 = 0; c0 < C1; c0 += 128) {
        const int c = c0 + lane * 4;
        if (c >= C1) break;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        int t = t0;
        for (; t + 3 < t1; t += 4) {                                              // four rows in flight, added in list order
            const int r0 = __ldg(lst + t), r1 = __ldg(lst + t + 1), r2 = __ldg(lst + t + 2), r3 = __ldg(lst + t + 3);
            const float4 d0 = g.get4(cloud * mk + r0, c), d1 = g.get4(cloud * mk + r1, c);
            const float4 d2 = g.get4(cloud * mk + r2, c), d3 = g.get4(cloud * mk + r3, c);
            acc.x += d0.x; acc.y += d0.y; acc.z += d0.z; acc.w += d0.w;
            acc.x += d1.x; acc.y += d1.y; acc.z += d1.z; acc.w += d1.w;
            acc.x += d2.x; acc.y += d2.y; acc.z += d2.z; acc.w += d2.w;
            acc.x += d3.x; acc.y += d3.y; acc.z += d3.z; acc.w += d3.w;
        }
        for (; t < t1; ++t) {
            const float4 d = g.get4(cloud * mk + __ldg(lst + t), c);
            acc.x += d.x; acc.y += d.y; acc.z += d.z; acc.w += d.w;
        }
        *reinterpret_cast<float4*>(dU + (size_t)pt * C1 + c) = acc;
    }
}

// ---- coordinate gradient of the fused first layer (psa_sa_conv1_bwd_xyz) ----
// One warp per query: groups of LPR lanes (4 channels per lane) take one grouped row each, RPW = 32 / LPR rows per step.  Each row
// gives v_r = W_xyz . dy0_r (three dot products over C1, lane partials in channel order, then a butterfly inside the group), stored
// as a float4 for the point-side pass; the query's dnew = -(v_0 + v_1 + ... ) is added in slot order by lane 0.  Fixed order.
template <int LPR>
__global__ void __launch_bounds__(256)
conv1_vxyz_kernel(const GradIn g, long long queries, int nsample, int C1, const float* __restrict__ w, float4* __restrict__ v,
                  float* __restrict__ dnew) {
    constexpr int RPW = 32 / LPR;
    const int lane = threadIdx.x & 31, sub = lane % LPR, rs = lane / LPR;
    const long long q = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (q >= queries) return;
    float sx = 0.f, sy = 0.f, sz = 0.f;                                     // lane 0: running slot-order sum of the query
    for (int k0 = 0; k0 < nsample; k0 += RPW) {
        const int k = k0 + rs;
        float ax = 0.f, ay = 0.f, az = 0.f;
        if (k < nsample) {
            const long long r = q * nsample + k;
            for (int c = 4 * sub; c < C1; c += 4 * LPR) {
                const float4 d = g.get4(r, c);
                const float4 wx = __ldg(reinterpret_cast<const float4*>(w + c));
                const float4 wy = __ldg(reinterpret_cast<const float4*>(w + C1 + c));
                const float4 wz = __ldg(reinterpret_cast<const float4*>(w + 2 * C1 + c));
                ax = fmaf(wx.w, d.w, fmaf(wx.z, d.z, fmaf(wx.y, d.y, fmaf(wx.x, d.x, ax))));
                ay = fmaf(wy.w, d.w, fmaf(wy.z, d.z, fmaf(wy.y, d.y, fmaf(wy.x, d.x, ay))));
                az = fmaf(wz.w, d.w, fmaf(wz.z, d.z, fmaf(wz.y, d.y, fmaf(wz.x, d.x, az))));
            }
        }
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) {
            ax += __shfl_xor_sync(0xffffffffu, ax, o);
            ay += __shfl_xor_sync(0xffffffffu, ay, o);
            az += __shfl_xor_sync(0xffffffffu, az, o);
        }
        if (sub == 0 && k < nsample) v[q * nsample + k] = make_float4(ax, ay, az, 0.f);
#pragma unroll
        for (int j = 0; j < RPW; ++j) {                                     // the step's rows, in slot order
            const float bx = __shfl_sync(0xffffffffu, ax, j * LPR), by = __shfl_sync(0xffffffffu, ay, j * LPR);
            const float bz = __shfl_sync(0xffffffffu, az, j * LPR);
            if (k0 + j < nsample) { sx += bx; sy += by; sz += bz; }
        }
    }
    if (lane == 0) { dnew[q * 3] = -sx; dnew[q * 3 + 1] = -sy; dnew[q * 3 + 2] = -sz; }
}

// dxyz[p] = sum of v over the rows that grouped point p, in ascending row order (the CSR of launch_group_csr); one thread per point
__global__ void __launch_bounds__(256)
point_vsum_csr_kernel(int n, int mk, long long total_points, const int* __restrict__ offsets, const int* __restrict__ list,
                      const float4* __restrict__ v, float* __restrict__ dxyz) {
    const long long pt = (long long)blockIdx.x * 256 + threadIdx.x;
    if (pt >= total_points) return;
    const long long cloud = pt / n;
    const int j = (int)(pt - cloud * n);
    const int* off = offsets + (size_t)cloud * (n + 1);
    const int* lst = list + (size_t)cloud * mk;
    const float4* vc = v + (size_t)cloud * mk;
    const int t0 = __ldg(off + j), t1 = __ldg(off + j + 1);
    float x = 0.f, y = 0.f, z = 0.f;
    int t = t0;
    for (; t + 3 < t1; t += 4) {                                            // four rows in flight, added in list order
        float4 d[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) d[u] = __ldg(vc + __ldg(lst + t + u));
#pragma unroll
        for (int u = 0; u < 4; ++u) { x += d[u].x; y += d[u].y; z += d[u].z; }
    }
    for (; t < t1; ++t) {
        const float4 d = __ldg(vc + __ldg(lst + t));
        x += d.x; y += d.y; z += d.z;
    }
    dxyz[pt * 3] = x; dxyz[pt * 3 + 1] = y; dxyz[pt * 3 + 2] = z;
}

// ---- bias gradient of a layer WITHOUT batch norm: db[c] = sum_r dy[r][c]; block = one column of one group of group_rows rows (a single
// group of all rows for the bias), fixed-order tree: db[grp][c] = sum over the group's rows ----
__global__ void __launch_bounds__(256) bias_grad_kernel(const GradIn g, long long group_rows, float* __restrict__ db) {
    __shared__ float red[256];
    const int c = blockIdx.x;
    const long long r0 = (long long)blockIdx.y * group_rows, r1 = r0 + group_rows;
    float t = 0.f;
    for (long long r = r0 + threadIdx.x; r < r1; r += 256) t += g.get(r, c);
    red[threadIdx.x] = t;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) db[(size_t)blockIdx.y * gridDim.x + c] = red[0];
}

// ---- loss ----
__global__ void softmax_xent_kernel(int b, int c, const float* __restrict__ logits, const int* __restrict__ labels, float* __restrict__ loss,
                                    float* __restrict__ dlogits) {
    __shared__ float rowloss[1024];
    const int r = threadIdx.x;
    if (r < b) {
        const float* l = logits + (size_t)r * c;
        float mx = l[0];
        for (int i = 1; i < c; ++i) mx = fmaxf(mx, l[i]);
        float se = 0.f;
        for (int i = 0; i < c; ++i) se += expf(l[i] - mx);
        const int lab = labels[r];
        // log(se) - (l[lab] - mx): both terms are of the loss's size.  (log(se) + mx) - l[lab] would round at the scale of the
        // logits, an error that grows with a common offset of the row that leaves the loss itself unchanged.
        rowloss[r] = logf(se) - (l[lab] - mx);
        const float invb = 1.f / (float)b;
        for (int i = 0; i < c; ++i) dlogits[(size_t)r * c + i] = (expf(l[i] - mx) / se - (i == lab ? 1.f : 0.f)) * invb;
    }
    __syncthreads();
    if (r == 0) {
        double s = 0.0;
        for (int i = 0; i < b; ++i) s += (double)rowloss[i];
        loss[0] = (float)(s / b);
    }
}

// ---- Adam ----
__global__ void adam_kernel(long long count, float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            float lr_t, float b1, float b2, float eps, float gscale) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
        const float gi = g[i] * gscale;
        const float mi = b1 * m[i] + (1.f - b1) * gi;
        const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
        m[i] = mi; v[i] = vi;
        p[i] -= lr_t * mi / (sqrtf(vi) + eps);
    }
}

constexpr long long kSmallM = 1024;        // rows up to this use the split-contraction path in forward / input gradient
static int small_m_splits(long long contraction) {
    long long s = contraction / 64;
    return (int)(s < 1 ? 1 : (s > 16 ? 16 : s));
}

int weight_grad_splits(long long rows, int tiles, long long* k_per_split) {
    long long want = (2LL * kNumSMs + tiles - 1) / tiles;
    long long maxs = (rows + 255) / 256;                       // at least 256 rows of contraction per split
    if (want > maxs) want = maxs;
    if (want < 1) want = 1;
    long long kps = (rows + want - 1) / want;
    kps = (kps + kGemmBK - 1) / kGemmBK * kGemmBK;
    *k_per_split = kps;
    return (int)((rows + kps - 1) / kps);
}

static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The GEMM launchers put the 128-row tiles of the output on gridDim.y
constexpr long long kMaxRowTiles = 65535;

// A psa_grad_in read by the training reductions (bn_bwd_partial, conv1_dwxyz_partial, group_grad_csr, conv1_vxyz).  Unlike the
// GEMM, they load it with GradIn's float4 / int4 accessors and have no scalar fallback, so every vector they read must be 16-byte
// aligned with rows a multiple of 4 floats, and the pooled routing must cover `rows` rows of `width` channels.  `read_y`: y is read
// whatever s / ca hold; `coeffs`: ca / cb / cc are read.
static int check_vec_grad(const char* fn, const psa_grad_in* g, long long rows, int width, bool read_y, bool coeffs) {
    PSA_REQUIRE(g->mode == 0 || g->mode == 1, "%s: grad_in mode %d (0 or 1)", fn, g->mode);
    if (read_y || g->s != nullptr || (coeffs && g->ca != nullptr))
        PSA_REQUIRE(g->y != nullptr && al16(g->y) && g->ld % 4 == 0, "%s: grad_in y must be 16-byte aligned with ld a multiple of 4 (ld=%lld)", fn,
                    g->ld);
    PSA_REQUIRE(al16(g->s) && al16(g->t), "%s: grad_in s / t must be 16-byte aligned", fn);
    if (coeffs) PSA_REQUIRE(al16(g->ca) && al16(g->cb) && al16(g->cc), "%s: grad_in ca / cb / cc must be 16-byte aligned", fn);
    if (g->mode == 0) {
        PSA_REQUIRE(g->dh != nullptr && al16(g->dh) && al16(g->mask) && g->ld_dh % 4 == 0,
                    "%s: grad_in dh / mask must be 16-byte aligned with ld_dh a multiple of 4 (ld_dh=%lld)", fn, g->ld_dh);
    } else {
        PSA_REQUIRE(g->C == width && g->pool_k >= 1 && rows % g->pool_k == 0,
                    "%s: pooled grad_in needs C == %d and pool_k dividing %lld rows (C=%d pool_k=%d)", fn, width, rows, g->C, g->pool_k);
        PSA_REQUIRE(g->dp != nullptr && g->pv != nullptr && g->argk != nullptr && al16(g->dp) && al16(g->pv) && al16(g->argk),
                    "%s: grad_in dp / pv / argk must be 16-byte aligned", fn);
    }
    return PSA_OK;
}

}  // namespace psa

using namespace psa;

extern "C" size_t psa_train_dense_workspace_bytes(long long rows, int K, int N) {
    // forward: (tiles_m, 2, N) statistics partials; weight gradient: (splits, K, N) partial products
    const size_t fwd = (size_t)((rows + 127) / 128) * 2 * (size_t)N * sizeof(float);
    const int bm = K <= 64 ? 64 : 128, bn = N <= 64 ? 64 : 128;
    const int tiles = ((K + bm - 1) / bm) * ((N + bn - 1) / bn);
    long long kps;
    const int splits = weight_grad_splits(rows, tiles, &kps);
    const size_t bwd = splits > 1 ? (size_t)splits * K * N * sizeof(float) : 0;
    // small-M forward / input-gradient products split their contraction: (splits <= 16, rows, max(K, N)) partial outputs
    const size_t small = rows <= kSmallM ? (size_t)16 * rows * (K > N ? K : N) * sizeof(float) : 0;
    size_t mx = fwd > bwd ? fwd : bwd;
    if (small > mx) mx = small;
    // tensor-core forward: statistics partials + the per-step weight image behind them
    if (tc_train_fwd_eligible(rows, K, N)) { const size_t tcw = ((fwd + 255) & ~(size_t)255) + tc_dense_image_bytes(K, N); if (tcw > mx) mx = tcw; }
    return mx + 256;
}

extern "C" int psa_train_dense_fwd(long long rows, int K, int N, const psa_act_in* in, const float* W, const float* bias, float* y,
                                   float* stats, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 0 && K >= 1 && N >= 1, "train_dense_fwd: bad dims rows=%lld K=%d N=%d", rows, K, N);
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(in && in->x && W && y, "train_dense_fwd: null buffer");
    cudaStream_t st = as_stream(stream);
    const long long tiles_m = (rows + 127) / 128;
    GemmOut o;
    o.out = y; o.ld_out = N; o.bias = bias; o.col_skip = 0; o.stat_partial = nullptr;
    if (stats != nullptr) {
        PSA_REQUIRE(workspace != nullptr && workspace_bytes >= (size_t)tiles_m * 2 * N * sizeof(float), "train_dense_fwd: workspace too small");
        o.stat_partial = reinterpret_cast<float*>(workspace);
    }
    // wide layers: wgmma path (bf16x3 operands, fp32 accumulate) when the input is a plain (rows, K) tensor without dropout
    if (tc_train_fwd_eligible(rows, K, N) && in->ld == K && in->mask == nullptr) {
        const size_t stat_bytes = ((size_t)tiles_m * 2 * N * sizeof(float) + 255) & ~(size_t)255;
        PSA_REQUIRE(workspace != nullptr && workspace_bytes >= stat_bytes + tc_dense_image_bytes(K, N), "train_dense_fwd: workspace too small");
        float* sp = stats ? reinterpret_cast<float*>(workspace) : nullptr;
        int rc0 = launch_tc_dense_train(rows, K, N, in->x, in->scale, in->shift, in->relu, W, bias, y, sp,
                                        reinterpret_cast<uint8_t*>(workspace) + stat_bytes, st);
        if (rc0 != PSA_OK) return rc0;
        if (stats != nullptr) return reduce_partials((int)tiles_m, 2 * N, sp, stats, st);
        return PSA_OK;
    }
    PSA_SUPPORTED(tiles_m <= kMaxRowTiles, "train_dense_fwd: rows=%lld exceeds %lld row tiles of 128 on the fp32 path", rows, kMaxRowTiles);
    const ActIn fa(*in);
    const MatIn fb{W, N};
    int rc;
    const int splits = rows <= kSmallM ? small_m_splits(K) : 1;
    if (splits > 1) {
        // few row tiles, long contraction (the FC head): split K over CTAs, finish in split order, statistics from the result
        PSA_REQUIRE(workspace != nullptr && workspace_bytes >= (size_t)splits * rows * N * sizeof(float), "train_dense_fwd: workspace too small");
        GemmOut po;
        po.out = reinterpret_cast<float*>(workspace); po.ld_out = N; po.bias = nullptr; po.col_skip = 0; po.stat_partial = nullptr;
        const long long kps = ((K + splits - 1) / splits + kGemmBK - 1) / kGemmBK * kGemmBK;
        const int nz = (int)((K + kps - 1) / kps);
        if (N <= 64) rc = launch_gemm<128, 64, true, true>(fa, fb, po, rows, N, K, nz, kps, st);
        else rc = launch_gemm<128, 128, true, true>(fa, fb, po, rows, N, K, nz, kps, st);
        if (rc != PSA_OK) return rc;
        const long long total = rows * N;
        splitk_finish_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(nz, rows, N, po.out, bias, y, N, 0);
        rc = check_launch("splitk_finish_kernel");
        if (rc != PSA_OK || stats == nullptr) return rc;
        col_stats_kernel<<<(N + 31) / 32, 1024, 0, st>>>(rows, N, y, stats);
        return check_launch("col_stats_kernel");
    }
    if (N <= 64) rc = launch_gemm<128, 64, true, true>(fa, fb, o, rows, N, K, 1, (long long)K + kGemmBK, st);
    else rc = launch_gemm<128, 128, true, true>(fa, fb, o, rows, N, K, 1, (long long)K + kGemmBK, st);
    if (rc != PSA_OK) return rc;
    if (stats != nullptr) return reduce_partials((int)tiles_m, 2 * N, o.stat_partial, stats, st);
    return PSA_OK;
}

extern "C" int psa_train_dense_fwd_grouped(long long rows, long long group_rows, int K, int N, const psa_act_in* in, const float* W,
                                           const float* bias, const float* group_add, float* y, float* stats, void* workspace,
                                           size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 0 && group_rows >= 1 && K >= 1 && N >= 1, "train_dense_fwd_grouped: bad dims rows=%lld group_rows=%lld K=%d N=%d",
                rows, group_rows, K, N);
    PSA_REQUIRE(rows % group_rows == 0, "train_dense_fwd_grouped: group_rows=%lld does not divide rows=%lld", group_rows, rows);
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(in && in->x && W && group_add && y, "train_dense_fwd_grouped: null buffer");
    cudaStream_t st = as_stream(stream);
    const long long tiles_m = (rows + 127) / 128;
    PSA_SUPPORTED(tiles_m <= kMaxRowTiles, "train_dense_fwd_grouped: rows=%lld exceeds %lld row tiles of 128", rows, kMaxRowTiles);
    GemmOut o;
    o.out = y; o.ld_out = N; o.bias = bias; o.col_skip = 0; o.stat_partial = nullptr;
    o.group_add = group_add; o.group_rows = group_rows;
    if (stats != nullptr) {
        PSA_REQUIRE(workspace != nullptr && workspace_bytes >= (size_t)tiles_m * 2 * N * sizeof(float), "train_dense_fwd_grouped: workspace too small");
        o.stat_partial = reinterpret_cast<float*>(workspace);
    }
    // one pass of the fp32 GEMM, the group rows added in its epilogue before the statistics
    const ActIn fa(*in);
    const MatIn fb{W, N};
    int rc;
    if (N <= 64) rc = launch_gemm<128, 64, true, true, true>(fa, fb, o, rows, N, K, 1, (long long)K + kGemmBK, st);
    else rc = launch_gemm<128, 128, true, true, true>(fa, fb, o, rows, N, K, 1, (long long)K + kGemmBK, st);
    if (rc != PSA_OK) return rc;
    if (stats != nullptr) return reduce_partials((int)tiles_m, 2 * N, o.stat_partial, stats, st);
    return PSA_OK;
}

extern "C" int psa_train_dense_bwd_input(long long rows, int K, int N, const psa_grad_in* g, const float* W, float* dx, long long ld_dx,
                                         int col_skip, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 0 && K >= 1 && N >= 1 && col_skip >= 0 && col_skip < K, "train_dense_bwd_input: bad dims");
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(g && W && dx, "train_dense_bwd_input: null buffer");
    PSA_SUPPORTED((rows + 127) / 128 <= kMaxRowTiles, "train_dense_bwd_input: rows=%lld exceeds %lld row tiles of 128", rows, kMaxRowTiles);
    GemmOut o;
    o.out = dx; o.ld_out = ld_dx; o.bias = nullptr; o.col_skip = col_skip; o.stat_partial = nullptr;
    const GradIn fa(*g);
    const MatIn fb{W, N};                                    // B(kc = n, col = k) = W[k][n]: contraction-contiguous
    cudaStream_t st = as_stream(stream);
    const int splits = rows <= kSmallM ? small_m_splits(N) : 1;
    if (splits > 1 && workspace != nullptr && workspace_bytes >= (size_t)splits * rows * K * sizeof(float)) {
        GemmOut po;
        po.out = reinterpret_cast<float*>(workspace); po.ld_out = K; po.bias = nullptr; po.col_skip = 0; po.stat_partial = nullptr;
        const long long kps = ((N + splits - 1) / splits + kGemmBK - 1) / kGemmBK * kGemmBK;
        const int nz = (int)((N + kps - 1) / kps);
        int rc;
        if (K <= 64) rc = launch_gemm<128, 64, true, false>(fa, fb, po, rows, K, N, nz, kps, st);
        else rc = launch_gemm<128, 128, true, false>(fa, fb, po, rows, K, N, nz, kps, st);
        if (rc != PSA_OK) return rc;
        const long long total = rows * K;
        splitk_finish_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(nz, rows, K, po.out, nullptr, dx, ld_dx, col_skip);
        return check_launch("splitk_finish_kernel");
    }
    if (K <= 64) return launch_gemm<128, 64, true, false>(fa, fb, o, rows, K, N, 1, (long long)N + kGemmBK, st);
    return launch_gemm<128, 128, true, false>(fa, fb, o, rows, K, N, 1, (long long)N + kGemmBK, st);
}

extern "C" int psa_train_dense_bwd_weight(long long rows, int K, int N, const psa_act_in* in, const psa_grad_in* g, float* dW,
                                          void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 1 && K >= 1 && N >= 1, "train_dense_bwd_weight: bad dims");
    PSA_REQUIRE(in && in->x && g && dW, "train_dense_bwd_weight: null buffer");
    cudaStream_t st = as_stream(stream);
    const int bm = K <= 64 ? 64 : 128, bn = N <= 64 ? 64 : 128;
    const int tiles = ((K + bm - 1) / bm) * ((N + bn - 1) / bn);
    long long kps;
    const int splits = weight_grad_splits(rows, tiles, &kps);
    GemmOut o;
    o.ld_out = N; o.bias = nullptr; o.col_skip = 0; o.stat_partial = nullptr;
    if (splits > 1) {
        PSA_REQUIRE(workspace != nullptr && workspace_bytes >= (size_t)splits * K * N * sizeof(float), "train_dense_bwd_weight: workspace too small");
        o.out = reinterpret_cast<float*>(workspace);
    } else {
        o.out = dW;
    }
    const ActIn fa(*in);
    const GradIn fb(*g);
    int rc;
    if (bm == 64 && bn == 64) rc = launch_gemm<64, 64, false, true>(fa, fb, o, K, N, rows, splits, kps, st);
    else if (bm == 64) rc = launch_gemm<64, 128, false, true>(fa, fb, o, K, N, rows, splits, kps, st);
    else if (bn == 64) rc = launch_gemm<128, 64, false, true>(fa, fb, o, K, N, rows, splits, kps, st);
    else rc = launch_gemm<128, 128, false, true>(fa, fb, o, K, N, rows, splits, kps, st);
    if (rc != PSA_OK) return rc;
    if (splits > 1) return reduce_partials(splits, K * N, o.out, dW, st);
    return PSA_OK;
}

extern "C" int psa_bn_finalize(int C, long long count, const float* stats, const float* gamma, const float* beta, float decay,
                               float* moving_mean, float* moving_var, float* scale, float* shift, float* mean_inv, psa_stream_t stream) {
    PSA_REQUIRE(C >= 1 && count >= 1 && stats && gamma && beta && scale && shift, "bn_finalize: bad arguments");
    bn_finalize_kernel<<<(C + 127) / 128, 128, 0, as_stream(stream)>>>(C, 1.0 / (double)count, stats, gamma, beta, decay, moving_mean, moving_var,
                                                                        scale, shift, mean_inv);
    return check_launch("bn_finalize_kernel");
}

extern "C" int psa_bn_finalize_rows(long long rows, int C, const float* y, const float* gamma, const float* beta, float decay,
                                    float* moving_mean, float* moving_var, float* scale, float* shift, float* mean_inv, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 1 && C >= 1 && y && gamma && beta && scale && shift, "bn_finalize_rows: bad arguments");
    bn_finalize_rows_kernel<<<(C + 31) / 32, 1024, 0, as_stream(stream)>>>(rows, C, y, gamma, beta, decay, moving_mean, moving_var, scale,
                                                                           shift, mean_inv);
    return check_launch("bn_finalize_rows_kernel");
}

extern "C" int psa_train_pool_fwd(long long groups, int pool_k, int C, const float* y, const float* scale, const float* shift, float* pooled,
                                  int* argk, psa_stream_t stream) {
    PSA_REQUIRE(groups >= 0 && pool_k >= 1 && C >= 4 && C % 4 == 0, "train_pool_fwd: C=%d must be a multiple of 4", C);
    if (groups == 0) return PSA_OK;
    PSA_REQUIRE(y && scale && shift && pooled && argk, "train_pool_fwd: null buffer");
    PSA_REQUIRE(al16(y) && al16(scale) && al16(shift) && al16(pooled) && al16(argk), "train_pool_fwd: y, scale, shift, pooled, argk must be 16-byte aligned");
    const long long total = groups * (C / 4);
    train_pool_fwd_kernel<<<(unsigned)((total + 127) / 128), 128, 0, as_stream(stream)>>>(
        groups, pool_k, C / 4, reinterpret_cast<const float4*>(y), reinterpret_cast<const float4*>(scale), reinterpret_cast<const float4*>(shift),
        reinterpret_cast<float4*>(pooled), reinterpret_cast<int4*>(argk));
    return check_launch("train_pool_fwd_kernel");
}

extern "C" int psa_pool_rows(long long groups, int pool_k, int C, int mode, const float* x, const float* dist, float* out, psa_stream_t stream) {
    PSA_REQUIRE(groups >= 0 && pool_k >= 1 && C >= 4 && C % 4 == 0, "pool_rows: C=%d must be a multiple of 4", C);
    PSA_REQUIRE(mode >= 0 && mode <= 2 && (mode != 2 || dist != nullptr), "pool_rows: mode %d", mode);
    if (groups == 0) return PSA_OK;
    PSA_REQUIRE(x && out, "pool_rows: null buffer");
    PSA_REQUIRE(al16(x) && al16(out), "pool_rows: x and out must be 16-byte aligned");
    const long long total = groups * (C / 4);
    pool_rows_kernel<<<(unsigned)((total + 127) / 128), 128, 0, as_stream(stream)>>>(groups, pool_k, C / 4, mode, reinterpret_cast<const float4*>(x), dist,
                                                                                       reinterpret_cast<float4*>(out));
    return check_launch("pool_rows_kernel");
}

static const int kBnbMaxBlocks = 4 * kNumSMs;

extern "C" size_t psa_bn_bwd_workspace_bytes(int C) { return (size_t)kBnbMaxBlocks * 2 * C * sizeof(float); }

extern "C" int psa_bn_bwd_coeffs(long long rows, int C, const psa_grad_in* g, const float* gamma, const float* mean_inv, float* dgamma,
                                 float* dbeta, float* ca, float* cb, float* cc, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 1 && C >= 4, "bn_bwd_coeffs: bad dims");
    PSA_SUPPORTED(C % 4 == 0 && C <= 1024, "bn_bwd_coeffs: C=%d must be a multiple of 4, at most 1024", C);
    PSA_REQUIRE(g && gamma && mean_inv && dgamma && dbeta && ca && cb && cc, "bn_bwd_coeffs: null buffer");
    PSA_REQUIRE(workspace && workspace_bytes >= psa_bn_bwd_workspace_bytes(C), "bn_bwd_coeffs: workspace too small");
    int rc = check_vec_grad("bn_bwd_coeffs", g, rows, C, true, false);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(al16(mean_inv), "bn_bwd_coeffs: mean_inv must be 16-byte aligned");
    cudaStream_t st = as_stream(stream);
    GradIn gi(*g);
    gi.ca = gi.cb = gi.cc = nullptr;
    // units the blocks iterate over: rows (dense dz) or pooled groups (max-pool routing)
    const long long units = gi.mode == 0 ? rows : rows / gi.pool_k;
    const int RL = kBnbThreads / (C / 4);
    long long blocks = (units + (long long)RL * 8 - 1) / ((long long)RL * 8);
    if (blocks > kBnbMaxBlocks) blocks = kBnbMaxBlocks;
    if (blocks < 1) blocks = 1;
    const long long upb = (units + blocks - 1) / blocks;
    blocks = (units + upb - 1) / upb;
    float* partial = reinterpret_cast<float*>(workspace);
    bn_bwd_partial_kernel<<<(unsigned)blocks, kBnbThreads, 0, st>>>(gi, units, C, mean_inv, upb, partial);
    rc = check_launch("bn_bwd_partial_kernel");
    if (rc != PSA_OK) return rc;
    return launch_bn_bwd_final((int)blocks, C, rows, partial, gamma, mean_inv, dgamma, dbeta, ca, cb, cc, st);
}

static size_t conv1_bwd_partial_bytes(int C1) { return ((size_t)kBnbMaxBlocks * 3 * C1 * sizeof(float) + 255) & ~(size_t)255; }
extern "C" size_t psa_sa_conv1_bwd_workspace_bytes(int b, int n, int m, int nsample, int C1, int want_dU) {
    size_t bytes = conv1_bwd_partial_bytes(C1);
    if (want_dU) bytes += ((size_t)b * (n + 1) + (size_t)b * m * nsample) * sizeof(int);     // CSR offsets + row lists
    return bytes;
}

extern "C" int psa_sa_conv1_bwd(int b, int n, int m, int nsample, int C1, const float* xyz, const float* new_xyz, const int* idx,
                                const psa_grad_in* g, float* dW_xyz, float* dU, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(b >= 1 && n >= 1 && m >= 1 && nsample >= 1, "sa_conv1_bwd: bad dims");
    PSA_SUPPORTED(C1 % 4 == 0 && C1 <= 1024, "sa_conv1_bwd: C1=%d", C1);
    PSA_REQUIRE(xyz && new_xyz && idx && g && dW_xyz, "sa_conv1_bwd: null buffer");
    PSA_REQUIRE(workspace && workspace_bytes >= psa_sa_conv1_bwd_workspace_bytes(b, n, m, nsample, C1, dU != nullptr), "sa_conv1_bwd: workspace too small");
    const long long rows = (long long)b * m * nsample;
    int rc = check_vec_grad("sa_conv1_bwd", g, rows, C1, false, true);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(al16(dU), "sa_conv1_bwd: dU must be 16-byte aligned");
    cudaStream_t st = as_stream(stream);
    const GradIn gi(*g);
    const int RL = kBnbThreads / (C1 / 4);
    long long blocks = (rows + (long long)RL * 8 - 1) / ((long long)RL * 8);
    if (blocks > kBnbMaxBlocks) blocks = kBnbMaxBlocks;
    const long long rpb = (rows + blocks - 1) / blocks;
    blocks = (rows + rpb - 1) / rpb;
    float* partial = reinterpret_cast<float*>(workspace);
    conv1_dwxyz_partial_kernel<<<(unsigned)blocks, kBnbThreads, 0, st>>>(gi, rows, nsample, (long long)m * nsample, n, m, C1, xyz, new_xyz, idx,
                                                                         rpb, partial);
    rc = check_launch("conv1_dwxyz_partial_kernel");
    if (rc != PSA_OK) return rc;
    rc = reduce_partials((int)blocks, 3 * C1, partial, dW_xyz, st);
    if (rc != PSA_OK) return rc;
    if (dU != nullptr) {
        // CSR scratch behind the dW partials: offsets (b, n+1) + list (b, m*nsample)
        uint8_t* wsb = reinterpret_cast<uint8_t*>(workspace) + conv1_bwd_partial_bytes(C1);
        int* offsets = reinterpret_cast<int*>(wsb);
        int* list = offsets + (size_t)b * (n + 1);
        rc = launch_group_csr(b, n, m * nsample, idx, offsets, list, st);
        if (rc != PSA_OK) return rc;
        const long long pts = (long long)b * n;
        group_grad_csr_kernel<<<(unsigned)((pts + 7) / 8), 256, 0, st>>>(gi, n, m * nsample, C1, pts, offsets, list, dU);
        return check_launch("group_grad_csr_kernel");
    }
    return PSA_OK;
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
extern "C" size_t psa_sa_conv1_bwd_xyz_workspace_bytes(int b, int n, int m, int nsample) {
    if (b <= 0 || n <= 0 || m <= 0 || nsample <= 0) return 256;
    const size_t rows = (size_t)b * m * nsample;
    // per-row v (float4) | CSR offsets (b, n+1) | row lists (b, m*nsample)
    return align256(rows * sizeof(float4)) + align256((size_t)b * (n + 1) * sizeof(int)) + rows * sizeof(int);
}

extern "C" int psa_sa_conv1_bwd_xyz(int b, int n, int m, int nsample, int C1, const float* W_xyz, const int* idx, const psa_grad_in* g,
                                    float* dxyz, float* dnew_xyz, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(b >= 1 && n >= 1 && m >= 1 && nsample >= 1, "sa_conv1_bwd_xyz: bad dims b=%d n=%d m=%d nsample=%d", b, n, m, nsample);
    PSA_REQUIRE((long long)m * nsample <= 0x7fffffffLL, "sa_conv1_bwd_xyz: m*nsample exceeds int32");
    PSA_SUPPORTED(C1 % 4 == 0 && C1 >= 4 && C1 <= 1024, "sa_conv1_bwd_xyz: C1=%d", C1);
    PSA_REQUIRE(W_xyz && idx && g && dxyz && dnew_xyz, "sa_conv1_bwd_xyz: null buffer");
    PSA_REQUIRE((reinterpret_cast<uintptr_t>(W_xyz) & 15) == 0, "sa_conv1_bwd_xyz: W_xyz must be 16-byte aligned");
    const size_t need = psa_sa_conv1_bwd_xyz_workspace_bytes(b, n, m, nsample);
    PSA_REQUIRE(workspace && workspace_bytes >= need, "sa_conv1_bwd_xyz: workspace of %zu bytes required, got %zu", need, workspace_bytes);
    PSA_REQUIRE(al16(workspace), "sa_conv1_bwd_xyz: workspace must be 16-byte aligned");
    const long long queries = (long long)b * m, rows = queries * nsample;
    int rc = check_vec_grad("sa_conv1_bwd_xyz", g, rows, C1, false, true);
    if (rc != PSA_OK) return rc;
    cudaStream_t st = as_stream(stream);
    const GradIn gi(*g);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    float4* v = reinterpret_cast<float4*>(ws);
    int* offsets = reinterpret_cast<int*>(ws + align256((size_t)rows * sizeof(float4)));
    int* list = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(offsets) + align256((size_t)b * (n + 1) * sizeof(int)));
    const unsigned qblocks = (unsigned)((queries + 7) / 8);
    if (C1 <= 32) conv1_vxyz_kernel<8><<<qblocks, 256, 0, st>>>(gi, queries, nsample, C1, W_xyz, v, dnew_xyz);
    else if (C1 <= 64) conv1_vxyz_kernel<16><<<qblocks, 256, 0, st>>>(gi, queries, nsample, C1, W_xyz, v, dnew_xyz);
    else conv1_vxyz_kernel<32><<<qblocks, 256, 0, st>>>(gi, queries, nsample, C1, W_xyz, v, dnew_xyz);
    rc = check_launch("conv1_vxyz_kernel");
    if (rc != PSA_OK) return rc;
    rc = launch_group_csr(b, n, m * nsample, idx, offsets, list, st);
    if (rc != PSA_OK) return rc;
    const long long pts = (long long)b * n;
    point_vsum_csr_kernel<<<(unsigned)((pts + 255) / 256), 256, 0, st>>>(n, m * nsample, pts, offsets, list, v, dxyz);
    return check_launch("point_vsum_csr_kernel");
}

extern "C" int psa_train_bias_grad(long long rows, int N, const psa_grad_in* g, float* db, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 1 && N >= 1 && g && db, "train_bias_grad: bad arguments");
    const GradIn gi(*g);
    bias_grad_kernel<<<N, 256, 0, as_stream(stream)>>>(gi, rows, db);
    return check_launch("bias_grad_kernel");
}

extern "C" int psa_train_bias_grad_grouped(long long rows, long long group_rows, int N, const psa_grad_in* g, float* db, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 1 && group_rows >= 1 && N >= 1 && g && db, "train_bias_grad_grouped: bad arguments");
    PSA_REQUIRE(rows % group_rows == 0, "train_bias_grad_grouped: group_rows=%lld does not divide rows=%lld", group_rows, rows);
    PSA_SUPPORTED(rows / group_rows <= 65535, "train_bias_grad_grouped: %lld groups (at most 65535)", rows / group_rows);
    const GradIn gi(*g);
    bias_grad_kernel<<<dim3((unsigned)N, (unsigned)(rows / group_rows)), 256, 0, as_stream(stream)>>>(gi, group_rows, db);
    return check_launch("bias_grad_kernel");
}

extern "C" int psa_softmax_xent(int b, int c, const float* logits, const int* labels, float* loss, float* dlogits, psa_stream_t stream) {
    PSA_REQUIRE(b >= 1 && c >= 1 && logits && labels && loss && dlogits, "softmax_xent: bad arguments");
    PSA_SUPPORTED(b <= 1024, "softmax_xent: batch %d > 1024", b);
    softmax_xent_kernel<<<1, ((b + 31) / 32) * 32, 0, as_stream(stream)>>>(b, c, logits, labels, loss, dlogits);
    return check_launch("softmax_xent_kernel");
}

extern "C" int psa_adam_step(long long count, float* params, const float* grads, float* m, float* v, float lr, float beta1, float beta2,
                             float eps, int step, float grad_scale, psa_stream_t stream) {
    PSA_REQUIRE(count >= 0 && step >= 1, "adam_step: bad arguments");
    if (count == 0) return PSA_OK;
    PSA_REQUIRE(params && grads && m && v, "adam_step: null buffer");
    const float lr_t = (float)((double)lr * sqrt(1.0 - pow((double)beta2, step)) / (1.0 - pow((double)beta1, step)));
    long long blocks = (count + 255) / 256;
    if (blocks > 8 * kNumSMs) blocks = 8 * kNumSMs;
    adam_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(count, params, grads, m, v, lr_t, beta1, beta2, eps, grad_scale);
    return check_launch("adam_kernel");
}
