// mfv.cu -- 3DmFV-Net's modified Fisher vector (3DmFV-Net/utils/tf_util.py:578-652), its dense 3-D convolutions
// (tf_util.conv3d, :254-311, SAME, stride 1, folded batch norm + ReLU) and its two pools (:406-429 max_pool3d, avg_pool3d), inference.
//
//   fisher_vector_kernel   one block per cloud: the (b, G, 20) Fisher vector, power- and L2-normalised, with every per-(point,
//                          Gaussian) term and every reduction in fp64 and in a fixed order.  Nothing of size b*n*G exists.
//   conv3d_tapmask_kernel  per 128-row tile, the kernel taps that reach inside the grid for at least one row of the tile
//   tc_conv3d_kernel       one conv layer as a GEMM over the b*r^3 voxel rows, K = k^3 * c in (tap, channel) order: the producer
//                          warps gather each 64-channel block of one tap's neighbour rows with cp.async (a neighbour outside the
//                          grid, or a row past the end, is zero-filled), a tile skips every tap outside the grid for all its rows,
//                          and the tap loop of a tile is split across CTAs whose partials a second kernel adds in a fixed order.
//                          Same ring, operand split and fp16x2 range guard as tc_spider_kernel (spider.cu).
//   conv3d_fma_kernel      the same layer on the fp32 FMA pipe (mode 1, and shapes the tensor path does not take: c = 20)
//   pool3d_*_kernel        the SAME 3^3 stride-1 average (divided by the in-grid count) and the SAME 2^3 stride-2 max
//
// Row order of every grid activation: voxel-major, row = voxel * b + cloud, voxel = (d * r + h) * r + w.  A 128-row tile then
// covers 128 / b consecutive voxels of every cloud, so at b >= 32 a tile sees at most five voxels and most taps of a 5^3 kernel
// lie outside the grid for all of them.
#include <float.h>

#include "common.cuh"
#include "mlp_internal.cuh"
#include "tc_common.cuh"

namespace psa {

using namespace tc;

// ------------------------------------------------------------------------------------------------------------------
// Fisher vector.  q_pg = softmax_g(log w_g - sum_d log sigma_gd - 1/2 sum_d z_pgd^2), z = (x - mu) / sigma, shifted by its
// maximum over g: in exact arithmetic this is the reference's ratio w N(x) / sum_g w N(x).  Where the reference's fp32 densities
// all underflow (a point far from every Gaussian) the reference divides 0 by 0 and returns NaN; this kernel returns the finite
// limit.  The sums of q z and q (z^2 - 1) cancel for Gaussians inside a roughly symmetric cloud and the power normalisation's
// square root turns an absolute error e into about sqrt(e), so the terms and sums are evaluated in fp64.
// Block = one cloud, 512 threads.  Phase 1: per point the maximum and the normaliser over the G Gaussians.  Phase 2: warp w
// reduces the 20 statistics of Gaussians w, w + 16, ... over the points (lanes stride the points, then a butterfly).  Phase 3:
// per column the L2 norm over the Gaussians, reduced in a fixed order.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kFvThreads = 512, kFvCols = 20;

__host__ __device__ inline size_t fv_smem_bytes(int n, int G) {
    return ((size_t)2 * n + (size_t)G * kFvCols + (size_t)G * 7) * sizeof(double) + (size_t)n * 3 * sizeof(float);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_min_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__global__ void __launch_bounds__(kFvThreads) fisher_vector_kernel(int n, int G, const float* __restrict__ points,
                                                                   const float* __restrict__ w, const float* __restrict__ mu,
                                                                   const float* __restrict__ sigma, float* __restrict__ out) {
    extern __shared__ double fv_smem[];
    double* s_m = fv_smem;                        // (n) max_g of the log weight-density
    double* s_inv = s_m + n;                      // (n) 1 / sum_g exp(l - max)
    double* s_fv = s_inv + n;                     // (G, 20) power-normalised statistics
    double* s_lc = s_fv + (size_t)G * kFvCols;    // (G) log w - sum_d log sigma
    double* s_mu = s_lc + G;                      // (G, 3)
    double* s_rs = s_mu + (size_t)G * 3;          // (G, 3) 1 / sigma
    float* s_x = reinterpret_cast<float*>(s_rs + (size_t)G * 3);   // (n, 3)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, b = blockIdx.x;
    const float* xb = points + (size_t)b * n * 3;
    for (int e = tid; e < 3 * n; e += kFvThreads) s_x[e] = __ldg(xb + e);
    for (int g = tid; g < G; g += kFvThreads) {
        double lc = log((double)__ldg(w + g));
        for (int d = 0; d < 3; ++d) {
            const double sg = (double)__ldg(sigma + g * 3 + d);
            lc -= log(sg);
            s_mu[g * 3 + d] = (double)__ldg(mu + g * 3 + d);
            s_rs[g * 3 + d] = 1.0 / sg;
        }
        s_lc[g] = lc;
    }
    __syncthreads();
    auto logd = [&](int p, int g) {
        const double z0 = ((double)s_x[p * 3] - s_mu[g * 3]) * s_rs[g * 3];
        const double z1 = ((double)s_x[p * 3 + 1] - s_mu[g * 3 + 1]) * s_rs[g * 3 + 1];
        const double z2 = ((double)s_x[p * 3 + 2] - s_mu[g * 3 + 2]) * s_rs[g * 3 + 2];
        return s_lc[g] - 0.5 * (z0 * z0 + z1 * z1 + z2 * z2);
    };
    for (int p = tid; p < n; p += kFvThreads) {
        double m = -DBL_MAX;
        for (int g = 0; g < G; ++g) m = fmax(m, logd(p, g));
        double s = 0.0;
        for (int g = 0; g < G; ++g) s += exp(logd(p, g) - m);
        s_m[p] = m;
        s_inv[p] = 1.0 / s;
    }
    __syncthreads();
    const double dn = (double)n;
    for (int g = warp; g < G; g += kFvThreads / 32) {
        const double wg = (double)__ldg(w + g);
        double pmax = -DBL_MAX, psum = 0.0;
        double mmax[3], mmin[3], msum[3], smax[3], smin[3], ssum[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) { mmax[d] = smax[d] = -DBL_MAX; mmin[d] = smin[d] = DBL_MAX; msum[d] = ssum[d] = 0.0; }
        for (int p = lane; p < n; p += 32) {
            const double q = exp(logd(p, g) - s_m[p]) * s_inv[p];
            pmax = fmax(pmax, q - wg);
            psum += q - wg;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const double z = ((double)s_x[p * 3 + d] - s_mu[g * 3 + d]) * s_rs[g * 3 + d];
                const double a = q * z, c = q * (z * z - 1.0);
                mmax[d] = fmax(mmax[d], a); mmin[d] = fmin(mmin[d], a); msum[d] += a;
                smax[d] = fmax(smax[d], c); smin[d] = fmin(smin[d], c); ssum[d] += c;
            }
        }
        double v[kFvCols];
        v[0] = warp_max_d(pmax);
        v[1] = warp_sum_d(psum);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            v[2 + d] = warp_max_d(mmax[d]); v[5 + d] = warp_min_d(mmin[d]); v[8 + d] = warp_sum_d(msum[d]);
            v[11 + d] = warp_max_d(smax[d]); v[14 + d] = warp_min_d(smin[d]); v[17 + d] = warp_sum_d(ssum[d]);
        }
        if (lane == 0) {
            const double fpi = 1.0 / (sqrt(wg) * dn), fmu = 1.0 / (dn * sqrt(wg)), fsg = 1.0 / (dn * sqrt(2.0 * wg));
#pragma unroll
            for (int i = 0; i < kFvCols; ++i) {
                const double t = v[i] * (i < 2 ? fpi : i < 11 ? fmu : fsg);
                s_fv[g * kFvCols + i] = copysign(sqrt(fabs(t)), t);
            }
        }
    }
    __syncthreads();
    for (int col = warp; col < kFvCols; col += kFvThreads / 32) {
        double ss = 0.0;
        for (int g = lane; g < G; g += 32) ss += s_fv[g * kFvCols + col] * s_fv[g * kFvCols + col];
        const double inv = 1.0 / sqrt(fmax(warp_sum_d(ss), 1e-12));
        for (int g = lane; g < G; g += 32) out[((size_t)b * G + g) * kFvCols + col] = (float)(s_fv[g * kFvCols + col] * inv);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// conv3d: tap activity per tile
// ------------------------------------------------------------------------------------------------------------------
constexpr int kMaskWords = 4;          // k^3 <= 125 taps -> four 32-bit words per tile

// does tap (oz, oy, ox) (offsets from the centre) reach inside the r^3 grid for some row of rows [row0, row1]?
__host__ __device__ inline bool conv_tap_active(long long row0, long long row1, int b, int r, int oz, int oy, int ox) {
    for (long long v = row0 / b; v <= row1 / b; ++v) {
        const int z = (int)(v / (r * r)), y = (int)(v / r % r), x = (int)(v % r);
        if (z + oz >= 0 && z + oz < r && y + oy >= 0 && y + oy < r && x + ox >= 0 && x + ox < r) return true;
    }
    return false;
}

__global__ void conv3d_tapmask_kernel(long long rows, int b, int r, int k, int ntiles, uint32_t* __restrict__ mask) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ntiles * kMaskWords) return;
    const int tile = e / kMaskWords, word = e % kMaskWords, h = k / 2;
    const long long row0 = (long long)tile * 128, row1 = min(rows, row0 + 128) - 1;
    uint32_t bits = 0;
    for (int bit = 0; bit < 32; ++bit) {
        const int tap = word * 32 + bit;
        if (tap < k * k * k && conv_tap_active(row0, row1, b, r, tap / (k * k) - h, tap / k % k - h, tap % k - h)) bits |= 1u << bit;
    }
    mask[e] = bits;
}

// the first tap at or after `from` set in a tile's mask words m, or 128
__device__ __forceinline__ int mask_next_g(const uint32_t* m, int from) {
    for (int wd = from >> 5; wd < kMaskWords; ++wd) {
        const uint32_t bits = __ldg(m + wd) & (wd == (from >> 5) ? 0xffffffffu << (from & 31) : 0xffffffffu);
        if (bits) return wd * 32 + __ffs(bits) - 1;
    }
    return 128;
}

// ------------------------------------------------------------------------------------------------------------------
// tc_conv3d_kernel<NP, NC>: out (rows, N) = relu((A . W) * scale + shift) over work units (128-row tile, 64 NC-column tile,
// split), persistent with a static unit order.  A[row][(tap, ch)] = x[neighbour(row, tap)][ch], or 0 outside the grid.  Unit
// (tile, nt, sp) takes the active K blocks [nact sp / S, nact (sp + 1) / S) of its tile, in (tap, channel block) order; with
// S > 1 it writes its partial (unscaled) to partial[sp] and conv3d_finalize_kernel adds the S partials in split order.
// CTA = two consumer warpgroups (rows 0-63 / 64-127) + a producer warpgroup whose four warps each gather 32 rows of every block
// while warp 0 also drops the block's weights in by TMA.  The consumers' K loop is tc_spider_kernel's.
// ------------------------------------------------------------------------------------------------------------------
struct Conv3dArgs {
    long long rows;            // b * r^3
    int b, r, k, c, N, Np;     // Np: N padded to the tile width (the image's width)
    int splits, KC;            // KC = k^3 * c / 64, the image's K blocks
    const float* x;            // (rows, ldx), 16-byte aligned, ldx % 4 == 0
    long long ldx;
    const uint32_t* tapmask;   // (tiles, 4)
    const uint8_t* image;      // W (k^3 c, Np) in the format of NP, tile width 64 NC
    const float* scale;        // (N) or null
    const float* shift;        // (N)
    int relu;
    float* out;                // row stride ldo
    long long ldo;
    float* partial;            // (splits, rows, Np) when splits > 1
    unsigned int* ovf = nullptr;
    const unsigned int* run_if = nullptr;
    const unsigned int* wflag = nullptr;
    const float* colscale = nullptr;
};

constexpr int kConvThreads = 384, kConvConsumers = 256;
constexpr uint32_t kConvXRow = 64u * 4u + 32u;
constexpr uint32_t kConvXBytes = 128u * kConvXRow;
constexpr uint32_t kConvRingBudget = 206u * 1024u;
__host__ __device__ constexpr uint32_t conv_stage_bytes(int NP, int NC) { return tc_block_bytes(64 * NC, NP) + kConvXBytes; }
__host__ __device__ constexpr int conv_stages(int NP, int NC) {
    return kConvRingBudget / conv_stage_bytes(NP, NC) < 4u ? (int)(kConvRingBudget / conv_stage_bytes(NP, NC)) : 4;
}

__device__ __forceinline__ void cp_async16_zfill(uint32_t smem_dst, const void* gmem_src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_dst), "l"(gmem_src), "r"(src_bytes) : "memory");
}

template <int NP, int NC>
__global__ void __launch_bounds__(kConvThreads, 1)
tc_conv3d_kernel(const __grid_constant__ Conv3dArgs a) {
    if (a.run_if != nullptr && *a.run_if == 0u) return;
    constexpr int Nt = 64 * NC, S = conv_stages(NP, NC);
    constexpr uint32_t bb = tc_block_bytes(Nt, NP), piece = Nt * 128u, SB = conv_stage_bytes(NP, NC);
    static_assert(S >= 2, "the ring needs two stages");
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_full[S], s_empty[S];
    __shared__ int s_zyx[128], s_cl[128];                           // the tile's rows: packed voxel coordinates (-1: past the end), cloud
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int CB = a.c / 64, NTC = a.Np / Nt, h = a.k / 2;
    const long long tiles = (a.rows + 127) / 128, nunits = tiles * NTC * a.splits;
    if (tid == 0) {
        for (int i = 0; i < S; ++i) { mbar_init(&s_full[i], 1 + 128); mbar_init(&s_empty[i], kConvConsumers / 32); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp >= kConvConsumers / 32) {
        // ---- producers: warp pw gathers tile rows [32 pw, 32 pw + 32) ----
        // 168 registers per thread at launch: the 128 x 128 the producers release are exactly the consumers' 256 x 64
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
        const int pw = warp - kConvConsumers / 32;
        uint32_t q = 0;
        // (32-bit unit and row indices, rows < 2^31; the tile's mask re-read from L1 as the tap advances: 40 registers)
        for (int unit = blockIdx.x; unit < (int)nunits; unit += gridDim.x) {
            const int sp = unit % a.splits, nt = unit / a.splits % NTC, tile = unit / a.splits / NTC, row0 = tile * 128;
            const uint32_t* tm = a.tapmask + tile * kMaskWords;
            const int nact = (__popc(__ldg(tm)) + __popc(__ldg(tm + 1)) + __popc(__ldg(tm + 2)) + __popc(__ldg(tm + 3))) * CB;
            const int j0 = nact * sp / a.splits, j1 = nact * (sp + 1) / a.splits;
            if (j0 == j1) continue;
            __syncwarp();                                            // the previous unit's reads of s_zyx are done
            {
                const int R = row0 + 32 * pw + lane;
                int zyx = -1, cl = 0;
                if (R < (int)a.rows) {
                    const int v = R / a.b;
                    cl = R - v * a.b;
                    zyx = v / (a.r * a.r) << 16 | v / a.r % a.r << 8 | v % a.r;
                }
                s_zyx[32 * pw + lane] = zyx;
                s_cl[32 * pw + lane] = cl;
            }
            __syncwarp();
            int tap = -1;
            for (int i = 0; i <= j0 / CB; ++i) tap = mask_next_g(tm, tap + 1);
            int chunk = j0 % CB;
            for (int j = j0; j < j1; ++j, ++q) {
                const int s = (int)(q % S);
                if (q >= (uint32_t)S) mbar_wait(&s_empty[s], ((q / S) - 1u) & 1u);
                if (pw == 0 && lane == 0) {
                    mbar_expect_tx(&s_full[s], bb);
                    const uint8_t* src = a.image + ((size_t)nt * a.KC + (size_t)tap * CB + chunk) * bb;
                    for (uint32_t o = 0; o < bb; o += 16384u) bulk_g2s(base + (uint32_t)s * SB + o, src + o, min(16384u, bb - o), &s_full[s]);
                }
                const int oz = tap / (a.k * a.k) - h, oy = tap / a.k % a.k - h, ox = tap % a.k - h;
                const int cc = (lane & 15) * 4, ch = chunk * 64 + cc;
                const uint32_t xs = smem_u32(base + (uint32_t)s * SB + bb);
                for (int rr = lane >> 4; rr < 32; rr += 2) {
                    const int row = 32 * pw + rr, zyx = s_zyx[row];
                    const int z = (zyx >> 16) + oz, y = ((zyx >> 8) & 255) + oy, x = (zyx & 255) + ox;
                    const bool in = zyx >= 0 && z >= 0 && z < a.r && y >= 0 && y < a.r && x >= 0 && x < a.r;
                    const float* src = in ? a.x + ((long long)((z * a.r + y) * a.r + x) * a.b + s_cl[row]) * a.ldx + ch : a.x;
                    cp_async16_zfill(xs + (uint32_t)row * kConvXRow + (uint32_t)cc * 4u, src, in ? 16u : 0u);
                }
                cp_async_mbar_arrive(&s_full[s]);
                if (++chunk == CB) { chunk = 0; tap = mask_next_g(tm, tap + 1); }
            }
        }
        return;
    }

    // ---- consumers: warp w holds tile rows 16w + g and 16w + g + 8 ----
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
    const int g = lane >> 2, t = lane & 3;
    uint32_t ovf = 0u;
    uint32_t q = 0;                                                 // ring uses
    for (long long unit = blockIdx.x; unit < nunits; unit += gridDim.x) {
        const int sp = (int)(unit % a.splits), nt = (int)(unit / a.splits % NTC);
        const long long tile = unit / a.splits / NTC, row0 = tile * 128;
        const uint32_t* tm = a.tapmask + tile * kMaskWords;
        const int nact = (__popc(__ldg(tm)) + __popc(__ldg(tm + 1)) + __popc(__ldg(tm + 2)) + __popc(__ldg(tm + 3))) * CB;
        const int nb = nact * (sp + 1) / a.splits - nact * sp / a.splits;
        const long long r[2] = {row0 + warp * 16 + g, row0 + warp * 16 + g + 8};

        // staged block of ring use u -> A fragments (out-of-grid neighbours and rows past the end were zero-filled)
        auto prep = [&](uint32_t (&A)[NP][4][4], uint32_t u) {
            const float* xs = reinterpret_cast<const float*>(base + (u % S) * SB + bb);
#pragma unroll
            for (int s = 0; s < 4; ++s)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int kl = 16 * s + 8 * hh + 2 * t;
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const float2 x = *reinterpret_cast<const float2*>(xs + (warp * 16 + g + 8 * i) * (int)(kConvXRow / 4) + kl);
                        uint32_t pc[NP];
                        split_pair<NP>(x.x, x.y, pc, ovf);
#pragma unroll
                        for (int e = 0; e < NP; ++e) A[e][s][i + 2 * hh] = pc[e];
                    }
                }
        };
        float acc[NC][32];
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
                if (c0 + CG == NC && kb + 1 < nb) {
                    mbar_wait(&s_full[(u + 1) % S], ((u + 1) / S) & 1u);
                    prep(An, u + 1);
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
        if (nb > 0) {
            uint32_t A0[NP][4][4], A1[NP][4][4];
            mbar_wait(&s_full[q % S], (q / S) & 1u);
            prep(A0, q);
            for (int kb = 0;; kb += 2) {
                step(A0, A1, q + kb, kb);
                if (kb + 1 == nb) break;
                step(A1, A0, q + kb + 1, kb + 1);
                if (kb + 2 == nb) break;
            }
            q += nb;
        } else {
#pragma unroll
            for (int c = 0; c < NC; ++c)
#pragma unroll
                for (int e = 0; e < 32; ++e) acc[c][e] = 0.f;
        }

        // ---- epilogue: fp16x2 column factor; the whole sum -> scale, shift, ReLU; a split's share -> its partial ----
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const int col = nt * Nt + c * 64 + 8 * jj + 2 * t;
                const float2 cs = NP == 2 ? __ldg(reinterpret_cast<const float2*>(a.colscale + col)) : make_float2(1.f, 1.f);
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    if (r[i] >= a.rows) continue;
                    float2 v = make_float2(acc[c][4 * jj + 2 * i] * cs.x, acc[c][4 * jj + 2 * i + 1] * cs.y);
                    if (a.splits > 1) {
                        *reinterpret_cast<float2*>(a.partial + ((size_t)sp * a.rows + r[i]) * a.Np + col) = v;
                    } else if (col < a.N) {
                        const float2 sh = __ldg(reinterpret_cast<const float2*>(a.shift + col));
                        if (a.scale != nullptr) {
                            const float2 sc = __ldg(reinterpret_cast<const float2*>(a.scale + col));
                            v = make_float2(fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y));
                        } else {
                            v = make_float2(v.x + sh.x, v.y + sh.y);
                        }
                        if (a.relu) v = make_float2(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f));
                        *reinterpret_cast<float2*>(a.out + (size_t)r[i] * a.ldo + col) = v;
                    }
                }
            }
    }
    if constexpr (NP == 2) {
        if (f16x2_overflowed(ovf) || (tid == 0 && a.wflag != nullptr && *a.wflag != 0u)) atomicOr(a.ovf, 1u);
    }
}

// out = relu(sum_sp partial[sp] * scale + shift), the partials added in split order
__global__ void conv3d_finalize_kernel(long long rows, int N, int Np, int splits, const float* __restrict__ partial,
                                       const float* __restrict__ scale, const float* __restrict__ shift, int relu, float* __restrict__ out,
                                       long long ldo) {
    const long long total = rows * N;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long row = e / N;
        const int col = (int)(e - row * N);
        float s = __ldg(partial + row * Np + col);
        for (int sp = 1; sp < splits; ++sp) s += __ldg(partial + ((size_t)sp * rows + row) * Np + col);
        float v = scale != nullptr ? fmaf(s, __ldg(scale + col), __ldg(shift + col)) : s + __ldg(shift + col);
        if (relu) v = fmaxf(v, 0.f);
        out[row * ldo + col] = v;
    }
}

// W (K, N) -> (K, Np), columns N..Np zero
__global__ void conv3d_pad_kernel(long long K, int N, int Np, const float* __restrict__ W, float* __restrict__ Wp) {
    const long long total = K * Np;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int col = (int)(e % Np);
        Wp[e] = col < N ? __ldg(W + e / Np * N + col) : 0.f;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// The same layer on the fp32 FMA pipe: 64 x 64 tiles, 256 threads of 4 x 4 outputs, K in steps of 16, every tap, each 64-wide
// K block summed on its own before it is added to the total (as the tensor path sums).
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) conv3d_fma_kernel(const __grid_constant__ Conv3dArgs a, const float* __restrict__ W) {
    __shared__ float As[16][64 + 4], Bs[16][64];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const long long row0 = (long long)blockIdx.x * 64;
    const int col0 = blockIdx.y * 64, K = a.k * a.k * a.k * a.c, h = a.k / 2;
    float tot[4][4] = {}, acc[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int e = tid + 256 * i, kr = e >> 6, rr = e & 63;
            const int kk = k0 + kr;
            const long long R = row0 + rr;
            float val = 0.f;
            if (kk < K && R < a.rows) {
                const int tap = kk / a.c, ch = kk - tap * a.c;
                const long long v = R / a.b;
                const int cl = (int)(R - v * a.b);
                const int z = (int)(v / (a.r * a.r)) + tap / (a.k * a.k) - h, y = (int)(v / a.r % a.r) + tap / a.k % a.k - h,
                          x = (int)(v % a.r) + tap % a.k - h;
                if (z >= 0 && z < a.r && y >= 0 && y < a.r && x >= 0 && x < a.r)
                    val = __ldg(a.x + ((long long)((z * a.r + y) * a.r + x) * a.b + cl) * a.ldx + ch);
            }
            As[kr][rr] = val;
            const int col = col0 + rr;
            Bs[kr][rr] = (kk < K && col < a.N) ? __ldg(W + (size_t)kk * a.N + col) : 0.f;
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
                for (int jj = 0; jj < 4; ++jj) acc[i][jj] = fmaf(av[i], bv[jj], acc[i][jj]);
        }
        __syncthreads();
        if ((k0 & 63) == 48 || k0 + 16 >= K) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) { tot[i][jj] += acc[i][jj]; acc[i][jj] = 0.f; }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long R = row0 + ty * 4 + i;
        if (R >= a.rows) continue;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int col = col0 + tx * 4 + jj;
            if (col >= a.N) continue;
            float v = a.scale != nullptr ? fmaf(tot[i][jj], __ldg(a.scale + col), __ldg(a.shift + col)) : tot[i][jj] + __ldg(a.shift + col);
            if (a.relu) v = fmaxf(v, 0.f);
            a.out[R * a.ldo + col] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// pools (voxel-major rows, c channels)
// ------------------------------------------------------------------------------------------------------------------
// SAME 3^3 stride-1 average: the sum over the in-grid neighbours (fixed order) divided by their count (tf.nn.avg_pool3d)
__global__ void pool3d_avg_kernel(int b, int r, int c, const float* __restrict__ x, float* __restrict__ out) {
    const long long total = (long long)b * r * r * r * c;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int ch = (int)(e % c);
        const long long row = e / c, v = row / b;
        const int cl = (int)(row - v * b), z = (int)(v / (r * r)), y = (int)(v / r % r), xx = (int)(v % r);
        float s = 0.f;
        int cnt = 0;
        for (int dz = -1; dz <= 1; ++dz)
            for (int dy = -1; dy <= 1; ++dy)
                for (int dx = -1; dx <= 1; ++dx) {
                    const int Z = z + dz, Y = y + dy, X = xx + dx;
                    if (Z < 0 || Z >= r || Y < 0 || Y >= r || X < 0 || X >= r) continue;
                    s += __ldg(x + ((long long)((Z * r + Y) * r + X) * b + cl) * c + ch);
                    ++cnt;
                }
        out[e] = s / (float)cnt;
    }
}

// SAME 2^3 stride-2 max: output grid ro = ceil(r / 2), the padding at the far end (TF puts the odd pad cell after)
__global__ void pool3d_max_kernel(int b, int r, int c, const float* __restrict__ x, float* __restrict__ out) {
    const int ro = (r + 1) / 2;
    const long long total = (long long)b * ro * ro * ro * c;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int ch = (int)(e % c);
        const long long row = e / c, v = row / b;
        const int cl = (int)(row - v * b), z = (int)(v / (ro * ro)), y = (int)(v / ro % ro), xx = (int)(v % ro);
        float m = -INFINITY;
        for (int dz = 0; dz < 2; ++dz)
            for (int dy = 0; dy < 2; ++dy)
                for (int dx = 0; dx < 2; ++dx) {
                    const int Z = 2 * z + dz, Y = 2 * y + dy, X = 2 * xx + dx;
                    if (Z >= r || Y >= r || X >= r) continue;
                    m = fmaxf(m, __ldg(x + ((long long)((Z * r + Y) * r + X) * b + cl) * c + ch));
                }
        out[e] = m;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------------------------
// the shapes the tensor path takes (the pointers' alignment is checked separately, conv_tc_aligned)
static bool conv_tc_shape(int c, int N) { return c % 64 == 0 && N % 32 == 0; }
// cp.async reads x in 16-byte chunks; the epilogue reads scale / shift and writes out in float2
static bool conv_tc_aligned(const float* x, long long ldx, const float* scale, const float* shift, const float* out, long long ldo) {
    auto al = [](const void* p, uintptr_t m) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & m) == 0; };
    return ldx % 4 == 0 && ldo % 2 == 0 && al(x, 15) && al(out, 7) && al(scale, 7) && al(shift, 7);
}

struct ConvPlan {
    int Nt, Np, splits;
    long long tiles;
    size_t mask, wpad, img, partial, total;
};
static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
// Tile width: 128 when Np allows it and the 128-wide tiles alone fill more than half of the SMs.  Splits: as many as keep
// tiles * column tiles * splits within one wave, at most 16, and at most half the K blocks a tile can have active.
// Workspace for np weight pieces (tc_np()): np = 3 holds the bf16x3 image; np = 2 holds the fp16x2 image, and the bf16x3 image of
// the guarded rerun in the same bytes (the rerun builds it after the fp16x2 launch, which is the image's last reader, has run).
static ConvPlan conv_plan(int b, int r, int k, int c, int N, int np) {
    ConvPlan p{};
    const long long rows = (long long)b * r * r * r;
    p.tiles = (rows + 127) / 128;
    p.Np = (N + 63) / 64 * 64;
    p.Nt = p.Np % 128 == 0 && 2 * p.tiles * (p.Np / 128) > kNumSMs ? 128 : 64;
    const long long units = p.tiles * (p.Np / p.Nt);
    const int reach = k < 2 * r - 1 ? k : 2 * r - 1;
    const long long maxk = (long long)reach * reach * reach * (c / 64);
    long long s = units >= kNumSMs ? 1 : kNumSMs / units;
    s = s < 16 ? s : 16;
    s = s < maxk / 2 ? s : (maxk / 2 > 1 ? maxk / 2 : 1);
    p.splits = (int)s;
    const long long K = (long long)k * k * k * c;
    size_t off = 256;                                        // word 0: range flag of the fp16x2 launch
    p.mask = off; off += al256((size_t)p.tiles * kMaskWords * 4);
    if (p.Np != N) { p.wpad = off; off += al256((size_t)K * p.Np * 4); }
    const size_t img3 = tc_image_alloc_bytes((int)K, p.Np, 3), img2 = tc_image_alloc_bytes((int)K, p.Np, 2);
    p.img = off; off += np == 2 && img2 > img3 ? img2 : img3;
    if (p.splits > 1) { p.partial = off; off += al256((size_t)p.splits * rows * p.Np * 4); }
    p.total = off;
    return p;
}

template <int NP, int NC>
static int launch_conv_shape(const Conv3dArgs& a, cudaStream_t st) {
    const size_t smem = (size_t)conv_stages(NP, NC) * conv_stage_bytes(NP, NC) + 1024;
    PSA_CUDA(cudaFuncSetAttribute(tc_conv3d_kernel<NP, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0, sms = 0;
    PSA_CUDA(cudaGetDevice(&dev));
    PSA_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const long long units = (a.rows + 127) / 128 * (a.Np / (64 * NC)) * a.splits;
    tc_conv3d_kernel<NP, NC><<<(unsigned)(units < sms ? units : sms), kConvThreads, smem, st>>>(a);
    return check_launch("tc_conv3d_kernel");
}
template <int NP>
static int launch_conv_np(const Conv3dArgs& a, int Nt, cudaStream_t st) {
    return Nt == 128 ? launch_conv_shape<NP, 2>(a, st) : launch_conv_shape<NP, 1>(a, st);
}

}  // namespace psa

using namespace psa;

extern "C" int psa_fisher_vector(int b, int n, int G, const float* points, const float* w, const float* mu, const float* sigma,
                                 float* out, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 1 && G >= 1, "fisher_vector: bad dims b=%d n=%d G=%d", b, n, G);
    PSA_SUPPORTED(fv_smem_bytes(n, G) <= 220u * 1024u, "fisher_vector: n=%d points and G=%d Gaussians do not fit one block's shared memory", n, G);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(points && w && mu && sigma && out, "fisher_vector: null buffer");
    const size_t smem = fv_smem_bytes(n, G);
    PSA_CUDA(cudaFuncSetAttribute(fisher_vector_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fisher_vector_kernel<<<(unsigned)b, kFvThreads, smem, as_stream(stream)>>>(n, G, points, w, mu, sigma, out);
    return check_launch("fisher_vector_kernel");
}

extern "C" size_t psa_conv3d_workspace_bytes(int b, int r, int k, int c, int c_out) {
    if (b < 0 || r < 1 || (k != 1 && k != 3 && k != 5) || c < 1 || c_out < 1) return 0;
    if (mlp_mode() == 1 || !conv_tc_shape(c, c_out)) return 0;          // the fp32-FMA kernel needs none
    return conv_plan(b, r, k, c, c_out, tc_np()).total;
}

extern "C" int psa_conv3d_infer(int b, int r, int k, int c, int c_out, const float* x, long long ldx, const float* W, const float* scale,
                                const float* shift, int relu, float* out, long long ldo, void* workspace, size_t workspace_bytes,
                                psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && r >= 1 && c >= 1 && c_out >= 1, "conv3d: bad dims b=%d r=%d c=%d c_out=%d", b, r, c, c_out);
    PSA_REQUIRE(k == 1 || k == 3 || k == 5, "conv3d: k=%d must be 1, 3 or 5", k);
    PSA_REQUIRE((long long)b * r * r * r < (1LL << 31) && (long long)k * k * k * c <= (1LL << 30), "conv3d: too large");
    PSA_REQUIRE(ldx >= c && ldo >= c_out, "conv3d: row strides ldx=%lld ldo=%lld below the widths %d, %d", ldx, ldo, c, c_out);
    PSA_REQUIRE(r < 256, "conv3d: r=%d must be below 256", r);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(x && W && shift && out, "conv3d: null buffer");
    cudaStream_t st = as_stream(stream);
    Conv3dArgs a;
    a.rows = (long long)b * r * r * r; a.b = b; a.r = r; a.k = k; a.c = c; a.N = c_out; a.Np = c_out; a.splits = 1;
    a.KC = k * k * k * c / 64; a.x = x; a.ldx = ldx; a.tapmask = nullptr; a.image = nullptr; a.scale = scale; a.shift = shift;
    a.relu = relu ? 1 : 0; a.out = out; a.ldo = ldo; a.partial = nullptr;
    if (mlp_mode() == 1 || !conv_tc_shape(c, c_out) || !conv_tc_aligned(x, ldx, scale, shift, out, ldo)) {
        const dim3 grid((unsigned)((a.rows + 63) / 64), (unsigned)((c_out + 63) / 64));
        conv3d_fma_kernel<<<grid, 256, 0, st>>>(a, W);
        return check_launch("conv3d_fma_kernel");
    }
    const ConvPlan pl = conv_plan(b, r, k, c, c_out, tc_np());
    a.Np = pl.Np;
    PSA_REQUIRE(workspace != nullptr && workspace_bytes >= pl.total,
                "conv3d: workspace of %zu bytes required (psa_conv3d_workspace_bytes), got %zu", pl.total, workspace_bytes);
    PSA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "conv3d: workspace must be 256-byte aligned");
    uint8_t* wsb = reinterpret_cast<uint8_t*>(workspace);
    const int K = k * k * k * c;
    uint32_t* mask = reinterpret_cast<uint32_t*>(wsb + pl.mask);
    conv3d_tapmask_kernel<<<(unsigned)((pl.tiles * kMaskWords + 127) / 128), 128, 0, st>>>(a.rows, b, r, k, (int)pl.tiles, mask);
    int rc = check_launch("conv3d_tapmask_kernel");
    if (rc != PSA_OK) return rc;
    const float* wsrc = W;
    if (pl.Np != c_out) {
        float* wp = reinterpret_cast<float*>(wsb + pl.wpad);
        conv3d_pad_kernel<<<1024, 256, 0, st>>>(K, c_out, pl.Np, W, wp);
        rc = check_launch("conv3d_pad_kernel");
        if (rc != PSA_OK) return rc;
        wsrc = wp;
    }
    a.tapmask = mask;
    a.splits = pl.splits;
    a.partial = pl.splits > 1 ? reinterpret_cast<float*>(wsb + pl.partial) : nullptr;
    const int Nt = pl.Nt | image_flag(tc_np());
    uint8_t* img3 = wsb + pl.img;
    if (tc_np() == 3) {
        rc = build_image(K, K, pl.Np, Nt, wsrc, img3, st);
        if (rc != PSA_OK) return rc;
        a.image = img3;
        rc = launch_conv_np<3>(a, pl.Nt, st);
    } else {
        unsigned int* flag = reinterpret_cast<unsigned int*>(wsb);
        PSA_CUDA(cudaMemsetAsync(flag, 0, 256, st));
        uint8_t* img2 = wsb + pl.img;
        rc = build_image(K, K, pl.Np, Nt, wsrc, img2, st);
        if (rc != PSA_OK) return rc;
        a.image = img2; a.ovf = flag; a.wflag = image_trailer(img2, K, pl.Np); a.colscale = image_colscale(img2, K, pl.Np);
        rc = launch_conv_np<2>(a, pl.Nt, st);
        if (rc != PSA_OK) return rc;
        // guarded rerun on bf16x3 operands: its image and its launch are no-ops unless the fp16x2 pass raised the flag
        rc = build_image(K, K, pl.Np, pl.Nt | kImageBf16x3, wsrc, img3, st, flag);
        if (rc != PSA_OK) return rc;
        a.image = img3; a.ovf = nullptr; a.wflag = nullptr; a.colscale = nullptr; a.run_if = flag;
        rc = launch_conv_np<3>(a, pl.Nt, st);
    }
    if (rc != PSA_OK || pl.splits == 1) return rc;
    const long long total = a.rows * c_out;
    conv3d_finalize_kernel<<<(unsigned)min((total + 255) / 256, 8192LL), 256, 0, st>>>(a.rows, c_out, pl.Np, pl.splits, a.partial, scale, shift,
                                                                                     a.relu, out, ldo);
    return check_launch("conv3d_finalize_kernel");
}

extern "C" int psa_pool3d(int b, int r, int c, int kind, const float* x, float* out, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && r >= 1 && c >= 1, "pool3d: bad dims b=%d r=%d c=%d", b, r, c);
    PSA_REQUIRE(kind == 0 || kind == 1, "pool3d: kind=%d must be 0 (3^3 average, stride 1) or 1 (2^3 max, stride 2)", kind);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(x && out, "pool3d: null buffer");
    const int ro = kind == 0 ? r : (r + 1) / 2;
    const long long total = (long long)b * ro * ro * ro * c;
    const unsigned grid = (unsigned)min((total + 255) / 256, 8192LL);
    if (kind == 0) {
        pool3d_avg_kernel<<<grid, 256, 0, as_stream(stream)>>>(b, r, c, x, out);
        return check_launch("pool3d_avg_kernel");
    }
    pool3d_max_kernel<<<grid, 256, 0, as_stream(stream)>>>(b, r, c, x, out);
    return check_launch("pool3d_max_kernel");
}
