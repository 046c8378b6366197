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
//                          gathered row (two for c = 32).  Same ring, operand split and range guard as tc_dense_kernel (tc_mlp.cu).
//   spider_fma_kernel      the same product on the fp32 FMA pipe (mode 1, and shapes the tensor path does not take: layer 1, c = 3)
//   group_norm_*           per (cloud, group) mean and centred variance in fp64 -> the per-cloud affine (scale, shift)
//   topk_pool_kernel       the two largest values of relu(y * scale + shift) per (cloud, channel)
#include <float.h>

#include "common.cuh"
#include "mlp_internal.cuh"
#include "tc_common.cuh"

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
// tc_spider_kernel<NP, NC>: y (rows, N) = A . Wp + bias over 128-row x 64 NC-channel tiles, persistent (static tile order).
// CTA = two consumer warpgroups (rows 0-63 / 64-127) + a producer warpgroup whose four warps each gather 32 rows of every K
// block (cp.async, 16 bytes per copy) while warp 0 also drops the block's weights in by TMA.  Per tile a producer warp first
// copies its rows' k neighbour indices to shared memory, so the gathers of a block only wait on shared-memory reads.
// The consumers' K loop is tc_dense_kernel's: per block one wgmma group on the registers prepared under the previous one, the
// block's sum added to fp32 accumulators (no tensor-core accumulation over more than 64 K).
// ------------------------------------------------------------------------------------------------------------------
struct SpiderArgs {
    long long rows;            // b * n
    int n, c, k, T, K, N;      // K = k * T * c, a multiple of 64
    const float* feat;         // (rows, c), 16-byte aligned
    const int* idx;            // (rows, k)
    const float* g;            // (rows * k, T)
    const float* fs;           // (b, c) or null, 8-byte aligned on the tensor path
    const float* fu;
    const uint8_t* image;      // Wp in the format of NP, tile width 64 NC
    const float* bias;         // (N), 8-byte aligned on the tensor path
    float* y;                  // (rows, N), 8-byte aligned on the tensor path
    unsigned int* ovf = nullptr;            // np = 2: raised when an operand left the fp16 range or a weight is not finite
    const unsigned int* run_if = nullptr;   // non-null: no-op unless *run_if != 0
    const unsigned int* wflag = nullptr;
    const float* colscale = nullptr;
};

constexpr int kSpiderThreads = 384, kSpiderConsumers = 256;
constexpr uint32_t kSpiderXRow = 64u * 4u + 32u;          // as tc_dense_kernel: conflict-free fragment reads
constexpr uint32_t kSpiderXBytes = 128u * kSpiderXRow;
constexpr uint32_t kSpiderRingBudget = 206u * 1024u;
__host__ __device__ constexpr uint32_t spider_stage_bytes(int NP, int NC) { return tc_block_bytes(64 * NC, NP) + kSpiderXBytes; }
__host__ __device__ constexpr int spider_stages(int NP, int NC) {
    return kSpiderRingBudget / spider_stage_bytes(NP, NC) < 4u ? (int)(kSpiderRingBudget / spider_stage_bytes(NP, NC)) : 4;
}

template <int NP, int NC>
__global__ void __launch_bounds__(kSpiderThreads, 1)
tc_spider_kernel(const __grid_constant__ SpiderArgs a) {
    if (a.run_if != nullptr && *a.run_if == 0u) return;
    constexpr int Nt = 64 * NC, S = spider_stages(NP, NC);
    constexpr uint32_t bb = tc_block_bytes(Nt, NP), piece = Nt * 128u, SB = spider_stage_bytes(NP, NC);
    static_assert(S >= 2, "the ring needs two stages");
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_full[S], s_empty[S];
    __shared__ int s_tile[S];
    __shared__ int s_nbr[128 * kSpiderMaxK];                        // the tile's neighbour rows (global row index)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int KC = a.K / 64, NTC = a.N / Nt, seg = a.T * a.c;
    const long long ntiles = (a.rows + 127) / 128 * NTC;
    if (tid == 0) {
        for (int i = 0; i < S; ++i) { mbar_init(&s_full[i], 1 + 128); mbar_init(&s_empty[i], kSpiderConsumers / 32); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp >= kSpiderConsumers / 32) {
        // ---- producers: warp pw gathers tile rows [32 pw, 32 pw + 32) ----
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
        const int pw = warp - kSpiderConsumers / 32;
        uint32_t q = 0;
        for (long long tile = blockIdx.x;; tile += gridDim.x) {
            const bool done = tile >= ntiles;
            const long long row0 = tile / NTC * 128;
            const int nt = (int)(tile % NTC);
            const int r0 = 32 * pw, nr = done ? 0 : (int)max(0LL, min(32LL, a.rows - row0 - r0));
            if (!done) {
                __syncwarp();                                        // the previous tile's reads of s_nbr are done
                for (int e = lane; e < nr * a.k; e += 32) {
                    const int r = e / a.k;
                    const long long p = row0 + r0 + r;
                    s_nbr[(r0 + r) * kSpiderMaxK + (e - r * a.k)] = (int)(p / a.n * a.n) + __ldg(a.idx + p * a.k + (e - r * a.k));
                }
                __syncwarp();
            }
            for (int kb = 0; kb < KC; ++kb, ++q) {
                const int s = (int)(q % S);
                if (q >= (uint32_t)S) mbar_wait(&s_empty[s], ((q / S) - 1u) & 1u);
                if (pw == 0 && lane == 0) {
                    s_tile[s] = done ? -1 : (int)tile;
                    if (done) {
                        mbar_arrive1(&s_full[s]);
                    } else {
                        mbar_expect_tx(&s_full[s], bb);
                        const uint8_t* src = a.image + ((size_t)nt * KC + kb) * bb;
                        for (uint32_t o = 0; o < bb; o += 16384u) bulk_g2s(base + (uint32_t)s * SB + o, src + o, min(16384u, bb - o), &s_full[s]);
                    }
                }
                if (!done) {
                    // lane (row half, 16-byte chunk): the chunk's column of the block is fixed per lane, so is its (j, t, c)
                    const int cc = (lane & 15) * 4, kk = kb * 64 + cc;
                    const int j = kk / seg, rem = kk - j * seg, ch = rem - rem / a.c * a.c;
                    const uint32_t xs = smem_u32(base + (uint32_t)s * SB + bb);
                    for (int r = lane >> 4; r < nr; r += 2) {
                        const int row = r0 + r;
                        cp_async16(xs + (uint32_t)row * kSpiderXRow + (uint32_t)cc * 4u, a.feat + (size_t)s_nbr[row * kSpiderMaxK + j] * a.c + ch);
                    }
                }
                cp_async_mbar_arrive(&s_full[s]);
                if (done) break;
            }
            if (done) return;
        }
    }

    // ---- consumers: warp w holds tile rows 16w + g and 16w + g + 8 ----
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
    const int g = lane >> 2, t = lane & 3;
    uint32_t ovf = 0u;
    uint32_t q = 0;                                                 // ring uses
    for (;;) {
        mbar_wait(&s_full[q % S], (q / S) & 1u);
        const int tile = s_tile[q % S];
        if (tile < 0) break;
        const long long row0 = (long long)(tile / NTC) * 128;
        const int nt = tile % NTC;
        const long long r[2] = {row0 + warp * 16 + g, row0 + warp * 16 + g + 8};
        const bool v[2] = {r[0] < a.rows, r[1] < a.rows};
        const int cb[2] = {v[0] ? (int)(r[0] / a.n) * a.c : 0, v[1] ? (int)(r[1] / a.n) * a.c : 0};   // the rows' clouds

        // gathered block of ring use u -> A fragments: the previous layer's group norm + ReLU, times g_t(delta_pj); rows past
        // `rows` read as zero (their staged bytes are stale)
        auto prep = [&](uint32_t (&A)[NP][4][4], uint32_t u, int kb) {
            const float* xs = reinterpret_cast<const float*>(base + (u % S) * SB + bb);
            // c % 32 == 0: each 32-column half of the block lies in one (j, t) slice, channels ch0 ..
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int kk = kb * 64 + 32 * hf, j = kk / seg, rem = kk - j * seg, tt = rem / a.c, ch0 = rem - tt * a.c;
                float gv[2];
#pragma unroll
                for (int i = 0; i < 2; ++i) gv[i] = v[i] ? __ldg(a.g + (r[i] * a.k + j) * a.T + tt) : 0.f;
#pragma unroll
                for (int s = 2 * hf; s < 2 * hf + 2; ++s)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int kl = 16 * s + 8 * h + 2 * t, ch = ch0 + kl - 32 * hf;
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            float2 x = make_float2(0.f, 0.f);
                            if (v[i]) {
                                x = *reinterpret_cast<const float2*>(xs + (warp * 16 + g + 8 * i) * (int)(kSpiderXRow / 4) + kl);
                                if (a.fs != nullptr) {
                                    const float2 sc = __ldg(reinterpret_cast<const float2*>(a.fs + cb[i] + ch));
                                    const float2 sh = __ldg(reinterpret_cast<const float2*>(a.fu + cb[i] + ch));
                                    x.x = fmaxf(fmaf(x.x, sc.x, sh.x), 0.f);
                                    x.y = fmaxf(fmaf(x.y, sc.y, sh.y), 0.f);
                                }
                                x.x *= gv[i];
                                x.y *= gv[i];
                            }
                            uint32_t pc[NP];
                            split_pair<NP>(x.x, x.y, pc, ovf);
#pragma unroll
                            for (int e = 0; e < NP; ++e) A[e][s][i + 2 * h] = pc[e];
                        }
                    }
            }
        };
        float acc[NC][32];
        // tc_dense_kernel's step: issue block kb's group on A, prepare block kb + 1 into An while it runs, wait, release, add
        constexpr int CG = NP == 3 && NC == 2 ? 1 : NC;            // 64-channel chunks per group
        auto step = [&](const uint32_t (&A)[NP][4][4], uint32_t (&An)[NP][4][4], uint32_t u, int kb) {
            const uint32_t wb = smem_u32(base + (u % S) * SB);
#pragma unroll
            for (int c0 = 0; c0 < NC; c0 += CG) {
                float d[CG][32];
                wg_fence();
#pragma unroll
                for (int tt = 0; tt < Split<NP>::kTerms; ++tt)
#pragma unroll
                    for (int s = 0; s < 4; ++s)
#pragma unroll
                        for (int c = 0; c < CG; ++c)
                            wg_mma_rs<NP>(d[c], A[Split<NP>::a(tt)][s][0], A[Split<NP>::a(tt)][s][1], A[Split<NP>::a(tt)][s][2], A[Split<NP>::a(tt)][s][3],
                                          wg_desc(wb + Split<NP>::w(tt) * piece + (uint32_t)(c0 + c) * 8192u + (uint32_t)s * 32u), (tt | s) ? 1u : 0u);
                wg_commit();
                if (c0 + CG == NC && kb + 1 < KC) {
                    mbar_wait(&s_full[(u + 1) % S], ((u + 1) / S) & 1u);
                    prep(An, u + 1, kb + 1);
                }
                wg_wait_all();
                if (c0 + CG == NC) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive1(&s_empty[u % S]);
                }
#pragma unroll
                for (int c = 0; c < CG; ++c) {
                    wg_fence_acc(d[c]);
#pragma unroll
                    for (int e = 0; e < 32; ++e) acc[c0 + c][e] = kb ? acc[c0 + c][e] + d[c][e] : d[c][e];
                }
            }
        };
        {
            uint32_t A0[NP][4][4], A1[NP][4][4];
            prep(A0, q, 0);
            for (int kb = 0;; kb += 2) {
                step(A0, A1, q + kb, kb);
                if (kb + 1 == KC) break;
                step(A1, A0, q + kb + 1, kb + 1);
                if (kb + 2 == KC) break;
            }
        }
        q += KC;

        // ---- epilogue: fp16x2 column factor, bias; pre-group-norm y ----
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const int col = nt * Nt + c * 64 + 8 * jj + 2 * t;
                const float2 cs = NP == 2 ? __ldg(reinterpret_cast<const float2*>(a.colscale + col)) : make_float2(1.f, 1.f);
                const float2 bi = __ldg(reinterpret_cast<const float2*>(a.bias + col));
#pragma unroll
                for (int i = 0; i < 2; ++i)
                    if (v[i])
                        *reinterpret_cast<float2*>(a.y + (size_t)r[i] * a.N + col) =
                            make_float2(fmaf(acc[c][4 * jj + 2 * i], cs.x, bi.x), fmaf(acc[c][4 * jj + 2 * i + 1], cs.y, bi.y));
            }
    }
    if constexpr (NP == 2) {
        if (f16x2_overflowed(ovf) || (tid == 0 && a.wflag != nullptr && *a.wflag != 0u)) atomicOr(a.ovf, 1u);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// The same product on the fp32 FMA pipe, in the reference's K order (j, c, t): 64 x 64 tiles, 256 threads of 4 x 4 outputs,
// K in steps of 16, each 64-wide K block summed on its own before it is added to the total (as the tensor path sums).
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) spider_fma_kernel(const __grid_constant__ SpiderArgs a, const float* __restrict__ W) {
    __shared__ float As[16][64 + 4], Bs[16][64];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const long long row0 = (long long)blockIdx.x * 64;
    const int col0 = blockIdx.y * 64, ct = a.c * a.T;
    float tot[4][4] = {}, part[4][4] = {};
    for (int k0 = 0; k0 < a.K; k0 += 16) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int e = tid + 256 * i, kr = e >> 6, rr = e & 63;
            const int kk = k0 + kr;
            const long long p = row0 + rr;
            float val = 0.f;
            if (kk < a.K && p < a.rows) {
                const int j = kk / ct, rem = kk - j * ct, ch = rem / a.T, tt = rem - ch * a.T;
                const int b = (int)(p / a.n);
                float x = __ldg(a.feat + ((long long)b * a.n + __ldg(a.idx + p * a.k + j)) * a.c + ch);
                if (a.fs != nullptr) x = fmaxf(fmaf(x, __ldg(a.fs + b * a.c + ch), __ldg(a.fu + b * a.c + ch)), 0.f);
                val = x * __ldg(a.g + (p * a.k + j) * a.T + tt);
            }
            As[kr][rr] = val;
            const int col = col0 + rr;
            Bs[kr][rr] = (kk < a.K && col < a.N) ? __ldg(W + (size_t)kk * a.N + col) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kr = 0; kr < 16; ++kr) {
            float av[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { av[i] = As[kr][ty * 4 + i]; bv[i] = Bs[kr][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) part[i][jj] = fmaf(av[i], bv[jj], part[i][jj]);
        }
        __syncthreads();
        if ((k0 & 63) == 48 || k0 + 16 >= a.K) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) { tot[i][jj] += part[i][jj]; part[i][jj] = 0.f; }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long p = row0 + ty * 4 + i;
        if (p >= a.rows) continue;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int col = col0 + tx * 4 + jj;
            if (col < a.N) a.y[(size_t)p * a.N + col] = tot[i][jj] + __ldg(a.bias + col);
        }
    }
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
static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
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

template <int NP, int NC>
static int launch_spider_shape(const SpiderArgs& a, cudaStream_t st) {
    const size_t smem = (size_t)spider_stages(NP, NC) * spider_stage_bytes(NP, NC) + 1024;
    PSA_CUDA(cudaFuncSetAttribute(tc_spider_kernel<NP, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0, sms = 0;
    PSA_CUDA(cudaGetDevice(&dev));
    PSA_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const long long tiles = (a.rows + 127) / 128 * (a.N / (64 * NC));
    tc_spider_kernel<NP, NC><<<(unsigned)(tiles < sms ? tiles : sms), kSpiderThreads, smem, st>>>(a);
    return check_launch("tc_spider_kernel");
}
template <int NP>
static int launch_spider_np(const SpiderArgs& a, int Nt, cudaStream_t st) {
    return Nt == 128 ? launch_spider_shape<NP, 2>(a, st) : launch_spider_shape<NP, 1>(a, st);
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
    a.bias = bias; a.y = y; a.image = nullptr;
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
    uint8_t* img3 = wsb + ws.img3;
    if (tc_np() == 3) {
        rc = build_image(K, K, c_out, Nt | kImageBf16x3, wp, img3, st);
        if (rc != PSA_OK) return rc;
        a.image = img3;
        return launch_spider_np<3>(a, Nt, st);
    }
    unsigned int* flag = reinterpret_cast<unsigned int*>(wsb);
    PSA_CUDA(cudaMemsetAsync(flag, 0, 256, st));
    uint8_t* img2 = wsb + ws.img2;
    rc = build_image(K, K, c_out, Nt | kImageF16x2, wp, img2, st);
    if (rc != PSA_OK) return rc;
    a.image = img2; a.ovf = flag; a.wflag = image_trailer(img2, K, c_out); a.colscale = image_colscale(img2, K, c_out);
    rc = launch_spider_np<2>(a, Nt, st);
    if (rc != PSA_OK) return rc;
    // guarded rerun on bf16x3 operands: its image and its launch are no-ops unless the fp16x2 pass raised the flag
    rc = build_image(K, K, c_out, Nt | kImageBf16x3, wp, img3, st, flag);
    if (rc != PSA_OK) return rc;
    a.image = img3; a.ovf = nullptr; a.wflag = nullptr; a.colscale = nullptr; a.run_if = flag;
    return launch_spider_np<3>(a, Nt, st);
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
