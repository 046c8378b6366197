// edgeconv2_train.cu -- training mode of the two-layer EdgeConv of DGCNN's input transform net (dgcnn/models/transform_nets.py:18-27:
// get_edge_feature -> tconv1 -> tconv2 -> reduce_max over k), batch statistics over all E = b*n*k edges in both layers:
//
//   y1_ij = Q_i + P_nn(i,j)                      (layer 1 exactly as edgeconv_train.cu evaluates it: the same PQ, the same fp32 add)
//   h1_ij = relu(y1_ij * scale1 + shift1)
//   y2_ij = h1_ij . W2 + b2                      (C1 = 64 -> C2 = 128 per edge: a real product over E rows, on wgmma)
//   out_ic = max_j relu(y2_ij * scale2 + shift2)
//
// No per-edge tensor of either layer is kept in the forward: every pass rebuilds h1 from PQ (gathered from L2) straight into the
// A fragment of the wgmma and recomputes y2.  The backward keeps one per-edge buffer, dz1 (E, C1).
//
// Tiling: a unit is 64 consecutive centre points; block j of a unit is the m64 tile whose row r is edge (centre r, neighbour j).  The
// max over k is then an element-wise max over the k blocks of a unit, in registers, and the fragment of every block has the same
// (centre, channel) positions.  A CTA is one warpgroup and walks a fixed chunk of kE2Chunk units: every partial sum is indexed by
// chunk, never by CTA, and reduced in chunk order (bit-reproducible).
//
// Passes (each recomputes y2; the products run on bf16x3 operands, six MMAs per product -- Split<3> -- so that small backward values
// keep fp32 accuracy whatever their magnitude):
//   kE2Stats  per-chunk [sum y2 | sum y2^2]                                         -> psa_bn_finalize(C2, E)
//   kE2Pool   pooled (b*n, C2), mask (b*n, C2) = k-bit set of the edges reaching the max, ywin = y2 of the first of them
//   kE2Dw2    dW2 = sum_e h1_e^T dy2_e: h1^T and dy2^T staged as bf16 pieces in shared memory, product on wgmma (both operands from
//             shared memory), per-chunk partials
//   kE2Dh1    dh1 = dy2 . W2^T on wgmma (the D fragment of y2 is the A fragment of dy2), dz1 = dh1 [h1 > 0] -> (E, C1)
// dW2 and dh1 are separate passes: together they would hold h1, y2, dy2, dh1 and the dW2 accumulators (224 registers) at once.
// dy2 = ca2 dz2 + cb2 y2 + cc2 with dz2 = R_ic on the masked edges (R = dout / popcount(mask) where the max is positive, else 0); its
// batch-norm sums are point-sized (the winning value ywin), and layer 1's come from dz1.  The layer-1 tail is edge_layer_tail.
#include <limits.h>

#include "mlp_internal.cuh"
#include "tc_common.cuh"

namespace psa {
namespace {

using namespace tc;

constexpr int kE2C1 = 64, kE2C2 = 128;   // the widths the kernels are written for (the T-net's tconv1 / tconv2)
constexpr int kE2MaxK = 32;              // one 32-bit mask word per (centre, channel)
constexpr int kE2MaxCloud = 51200;       // points per cloud of the reverse neighbour lists (launch_group_csr)
constexpr int kE2Rows = 64;              // centres per unit = rows of a block
constexpr int kE2Chunk = 4;              // units per CTA, the index of every partial sum
constexpr int kE2Threads = 128;          // one warpgroup

enum { kE2Stats = 0, kE2Pool = 1, kE2Dw2 = 2, kE2Dh1 = 3 };

// bf16x3 images (3 pieces of [64][64] K-major SWIZZLE_128B per 64 x 64 block, blocks (n/64, k/64) in n-major order)
constexpr uint32_t kE2Piece = 64u * 128u;          // one piece of a 64 x 64 block
constexpr uint32_t kE2Block = 3u * kE2Piece;       // 24 KB
constexpr uint32_t kE2Image = 2u * kE2Block;       // C1 x C2 = two blocks
// shared memory (byte offsets from the 1 KB-aligned base)
constexpr uint32_t kE2SmemF = 0;                                 // image of W2 as B of y2 = h1 . W2   ([C2][C1])
constexpr uint32_t kE2SmemX = kE2Image;                          // kE2Dh1: image of W2^T as B of dh1 = dy2 . W2^T ([C1][C2])
constexpr uint32_t kE2SmemHt = kE2Image;                         // kE2Dw2: h1^T pieces, [C1][64 edges]
constexpr uint32_t kE2SmemDyt = kE2SmemHt + 3u * kE2Piece;       // kE2Dw2: dy2^T pieces, [C2][64 edges]
constexpr uint32_t kE2SmemAcc = kE2SmemDyt + 6u * kE2Piece;      // kE2Dw2: fp32 dW2 accumulators of the chunk
constexpr uint32_t kE2SmemVec = kE2SmemAcc + kE2C1 * kE2C2 * 4u; // per-channel vectors
__host__ __device__ constexpr uint32_t e2_smem_bytes(int mode) {
    return (mode == kE2Dw2 ? kE2SmemVec : kE2Image + (mode == kE2Dh1 ? kE2Image : 0u)) + 8u * kE2C2 * 4u + 4u * 2u * 64u * 4u + 1024u;
}

struct E2Args {
    long long points, units;
    int n, k;
    const float* PQ;       // (points, 2 C1) = [Q | P] of layer 1
    const int* nn;         // (points, k)
    const float* s1;       // layer-1 batch-norm affine (C1)
    const float* t1;
    const float* b2;       // (C2) or null
    const uint8_t* imgF;   // bf16x3 image of W2 as B of h1 . W2
    const uint8_t* imgX;   // bf16x3 image of W2^T as B of dy2 . W2^T
    const float* s2;       // layer-2 batch-norm affine (C2)
    const float* t2;
    const float* coef2;    // (3, C2) = ca2, cb2, cc2
    const float* R;        // (points, C2)
    float* part;           // per-chunk partials
    float* pooled;         // (points, C2)
    uint32_t* mask;
    float* ywin;
    float* dz1;            // (points * k, C1)
};

// element (k, n) of the (K, N) matrix at W[k * ldk + n * ldn] -> bf16x3 image of [N][K], 64 x 64 blocks
__global__ void edge2_image_kernel(int K, int N, int ldk, int ldn, const float* __restrict__ W, uint8_t* __restrict__ image) {
    const int KC = K / 64;
    uint32_t ovf = 0u;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < K * N; e += gridDim.x * blockDim.x) {
        const int n = e % N, k = e / N;
        uint32_t pc[3];
        split_pair<3>(__ldg(W + (size_t)k * ldk + (size_t)n * ldn), 0.f, pc, ovf);
        uint8_t* blk = image + (size_t)((n / 64) * KC + (k >> 6)) * kE2Block;
        const uint32_t off = swz_off_bf16(n % 64, k & 63, 64);
#pragma unroll
        for (int i = 0; i < 3; ++i) *reinterpret_cast<uint16_t*>(blk + i * kE2Piece + off) = (uint16_t)(pc[i] & 0xffffu);
    }
}

// Fragment positions: thread (warp w, g = lane / 4, t = lane % 4) holds, of a 64-channel half, element i = 4 jb + 2 hr + e:
// row 16 w + g + 8 hr, column 8 jb + 2 t + e.  The A fragment of a K = 64 product uses the same positions: pair (i, i + 1), e = 0,
// is register ((jb & 1) << 1) | hr of K step jb >> 1.
__device__ __forceinline__ int e2_row(int hr) { return ((threadIdx.x >> 5) << 4) + ((threadIdx.x & 31) >> 2) + 8 * hr; }
__device__ __forceinline__ int e2_col(int jb) { return 8 * jb + 2 * (threadIdx.x & 3); }

// h1 of block j of `unit` -> A pieces (and, when HT is set, the pieces of h1^T into shared memory); hpos bit i = [h1 > 0]
template <bool HT>
__device__ __forceinline__ void e2_build_h1(const E2Args& a, const float* __restrict__ s1, const float* __restrict__ t1, long long unit, int j,
                                            uint32_t (&A)[3][4][4], uint32_t& hpos, uint8_t* ht) {
    hpos = 0u;
    uint32_t ovf = 0u;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int r = e2_row(hr);
        const long long p = unit * kE2Rows + r;
        const bool valid = p < a.points;
        const float* q = a.PQ;
        const float* pn = a.PQ;
        if (valid) {
            const long long base = (p / a.n) * a.n;
            q += (size_t)p * 2 * kE2C1;
            pn += (size_t)(base + __ldg(a.nn + (size_t)p * a.k + j)) * 2 * kE2C1 + kE2C1;
        }
#pragma unroll
        for (int jb = 0; jb < 8; ++jb) {
            const int c = e2_col(jb);
            float h[2] = {0.f, 0.f};
            if (valid) {
                const float2 qv = __ldg(reinterpret_cast<const float2*>(q + c)), pv = __ldg(reinterpret_cast<const float2*>(pn + c));
                h[0] = fmaxf(fmaf(__fadd_rn(qv.x, pv.x), s1[c], t1[c]), 0.f);
                h[1] = fmaxf(fmaf(__fadd_rn(qv.y, pv.y), s1[c + 1], t1[c + 1]), 0.f);
            }
            const int i = 4 * jb + 2 * hr;
            hpos |= (h[0] > 0.f ? 1u << i : 0u) | (h[1] > 0.f ? 2u << i : 0u);
            uint32_t pc[3];
            split_pair<3>(h[0], h[1], pc, ovf);
#pragma unroll
            for (int pi = 0; pi < 3; ++pi) {
                A[pi][jb >> 1][((jb & 1) << 1) | hr] = pc[pi];
                if (HT) {
                    *reinterpret_cast<uint16_t*>(ht + pi * kE2Piece + swz_off_bf16(c, r, 64)) = (uint16_t)(pc[pi] & 0xffffu);
                    *reinterpret_cast<uint16_t*>(ht + pi * kE2Piece + swz_off_bf16(c + 1, r, 64)) = (uint16_t)(pc[pi] >> 16);
                }
            }
        }
    }
}

// D[64 x 64] = A[64 x 64] . B, B = the half-th 64 x 64 block pair of an image at smem address img (K step s at +32 B): 24 straight-line MMAs
__device__ __forceinline__ void e2_mma(float (&d)[32], const uint32_t (&A)[3][4][4], uint32_t img, uint32_t accumulate) {
    wg_fence();
#pragma unroll
    for (int tt = 0; tt < Split<3>::kTerms; ++tt)
#pragma unroll
        for (int s = 0; s < 4; ++s)
            wg_mma_rs<3>(d, A[Split<3>::a(tt)][s][0], A[Split<3>::a(tt)][s][1], A[Split<3>::a(tt)][s][2], A[Split<3>::a(tt)][s][3],
                         wg_desc(img + Split<3>::w(tt) * kE2Piece + (uint32_t)s * 32u), (accumulate | tt | s) ? 1u : 0u);
    wg_commit();
    wg_wait_all();
    wg_fence_acc(d);
}

// dy2 of the half's fragment (0 on rows past the last point)
__device__ __forceinline__ void e2_dy2(const E2Args& a, const float* __restrict__ coef, long long unit, int j, int half, float (&d)[32]) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const long long p = unit * kE2Rows + e2_row(hr);
        const bool valid = p < a.points;
#pragma unroll
        for (int jb = 0; jb < 8; ++jb) {
            const int c = 64 * half + e2_col(jb);
            uint2 m = make_uint2(0u, 0u);
            float2 r = make_float2(0.f, 0.f);
            if (valid) {
                m = __ldg(reinterpret_cast<const uint2*>(a.mask + (size_t)p * kE2C2 + c));
                r = __ldg(reinterpret_cast<const float2*>(a.R + (size_t)p * kE2C2 + c));
            }
            const int i = 4 * jb + 2 * hr;
            const float dz0 = (m.x >> j) & 1u ? r.x : 0.f, dz1 = (m.y >> j) & 1u ? r.y : 0.f;
            d[i] = valid ? fmaf(coef[c], dz0, fmaf(coef[kE2C2 + c], d[i], coef[2 * kE2C2 + c])) : 0.f;
            d[i + 1] = valid ? fmaf(coef[c + 1], dz1, fmaf(coef[kE2C2 + c + 1], d[i + 1], coef[2 * kE2C2 + c + 1])) : 0.f;
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(kE2Threads, 1) edge2_train_kernel(E2Args a) {
    extern __shared__ uint8_t e2_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(e2_raw) + 1023) & ~(uintptr_t)1023);
    __shared__ __align__(8) uint64_t bar;
    float* vec = reinterpret_cast<float*>(smem + (MODE == kE2Dw2 ? kE2SmemVec : kE2Image + (MODE == kE2Dh1 ? kE2Image : 0u)));
    float* s1 = vec;                       // C1
    float* t1 = vec + kE2C1;               // C1
    float* b2 = vec + 2 * kE2C1;           // C2
    float* v2 = b2 + kE2C2;                // s2, t2 (kE2Pool) or ca2, cb2, cc2 (backward): 3 C2
    float* red = v2 + 3 * kE2C2;           // kE2Stats: (4 warps, 2, 64)
    const uint32_t base = smem_u32(smem);
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (tid == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    for (int i = tid; i < kE2C1; i += kE2Threads) { s1[i] = __ldg(a.s1 + i); t1[i] = __ldg(a.t1 + i); }
    for (int i = tid; i < kE2C2; i += kE2Threads) {
        b2[i] = a.b2 != nullptr ? __ldg(a.b2 + i) : 0.f;
        if (MODE == kE2Pool) { v2[i] = __ldg(a.s2 + i); v2[kE2C2 + i] = __ldg(a.t2 + i); }
        if (MODE == kE2Dw2 || MODE == kE2Dh1)
            for (int q = 0; q < 3; ++q) v2[q * kE2C2 + i] = __ldg(a.coef2 + q * kE2C2 + i);
    }
    if (MODE == kE2Dw2)
        for (int i = tid; i < kE2C1 * kE2C2; i += kE2Threads) reinterpret_cast<float*>(smem + kE2SmemAcc)[i] = 0.f;
    __syncthreads();
    if (tid == 0) {
        const uint32_t bytes = kE2Image * (MODE == kE2Dh1 ? 2u : 1u);
        mbar_expect_tx(&bar, bytes);
        for (uint32_t o = 0; o < kE2Image; o += kE2Block) bulk_g2s(smem + kE2SmemF + o, a.imgF + o, kE2Block, &bar);
        if (MODE == kE2Dh1)
            for (uint32_t o = 0; o < kE2Image; o += kE2Block) bulk_g2s(smem + kE2SmemX + o, a.imgX + o, kE2Block, &bar);
    }
    mbar_wait(&bar, 0);

    const long long chunk = blockIdx.x, u0 = chunk * kE2Chunk;
    const long long u1 = u0 + kE2Chunk < a.units ? u0 + kE2Chunk : a.units;
    uint32_t A[3][4][4];
    uint32_t hpos;
    float d[32];

    if constexpr (MODE == kE2Stats || MODE == kE2Pool) {
        for (int half = 0; half < 2; ++half) {
            const uint32_t img = base + kE2SmemF + (uint32_t)half * kE2Block;
            float cs[16], cq[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) { cs[i] = 0.f; cq[i] = 0.f; }
            for (long long unit = u0; unit < u1; ++unit) {
                float mx[32], yw[32];
                uint32_t mk[32];
#pragma unroll
                for (int i = 0; i < 32; ++i) { mx[i] = -1.f; yw[i] = 0.f; mk[i] = 0u; }   // relu output >= 0: the first edge beats the sentinel
                for (int j = 0; j < a.k; ++j) {
                    e2_build_h1<false>(a, s1, t1, unit, j, A, hpos, nullptr);
                    e2_mma(d, A, img, 0u);
#pragma unroll
                    for (int i = 0; i < 32; ++i) {
                        const int c = 64 * half + e2_col(i >> 2) + (i & 1);
                        const bool valid = unit * kE2Rows + e2_row((i >> 1) & 1) < a.points;
                        const float y = d[i] + b2[c];
                        if (MODE == kE2Stats) {
                            if (valid) {
                                cs[((i >> 2) << 1) | (i & 1)] += y;
                                cq[((i >> 2) << 1) | (i & 1)] = fmaf(y, y, cq[((i >> 2) << 1) | (i & 1)]);
                            }
                        } else {
                            const float z = fmaxf(fmaf(y, v2[c], v2[kE2C2 + c]), 0.f);
                            if (z > mx[i]) { mx[i] = z; mk[i] = 1u << j; yw[i] = y; }
                            else if (z == mx[i]) mk[i] |= 1u << j;
                        }
                    }
                }
                if (MODE == kE2Pool) {
#pragma unroll
                    for (int hr = 0; hr < 2; ++hr) {
                        const long long p = unit * kE2Rows + e2_row(hr);
                        if (p >= a.points) continue;
#pragma unroll
                        for (int jb = 0; jb < 8; ++jb) {
                            const int i = 4 * jb + 2 * hr;
                            const size_t o = (size_t)p * kE2C2 + 64 * half + e2_col(jb);
                            *reinterpret_cast<float2*>(a.pooled + o) = make_float2(mx[i], mx[i + 1]);
                            *reinterpret_cast<uint2*>(a.mask + o) = make_uint2(mk[i], mk[i + 1]);
                            *reinterpret_cast<float2*>(a.ywin + o) = make_float2(yw[i], yw[i + 1]);
                        }
                    }
                }
            }
            if (MODE == kE2Stats) {
                // column sums of the chunk: across g (lane bits 2..4) in a fixed butterfly, then across the 4 warps in order
#pragma unroll
                for (int i = 0; i < 16; ++i) {
#pragma unroll
                    for (int m = 4; m <= 16; m <<= 1) {
                        cs[i] += __shfl_xor_sync(0xffffffffu, cs[i], m);
                        cq[i] += __shfl_xor_sync(0xffffffffu, cq[i], m);
                    }
                }
                if (lane < 4) {
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int c = 8 * (i >> 1) + 2 * lane + (i & 1);
                        red[(w * 2 + 0) * 64 + c] = cs[i];
                        red[(w * 2 + 1) * 64 + c] = cq[i];
                    }
                }
                __syncthreads();
                {
                    const int which = tid >> 6, c = tid & 63;
                    float s = 0.f;
#pragma unroll
                    for (int ww = 0; ww < 4; ++ww) s += red[(ww * 2 + which) * 64 + c];
                    a.part[(size_t)chunk * 2 * kE2C2 + which * kE2C2 + 64 * half + c] = s;
                }
                __syncthreads();
            }
        }
    } else if constexpr (MODE == kE2Dw2) {
        uint8_t* ht = smem + kE2SmemHt;
        uint8_t* dyt = smem + kE2SmemDyt;
        float* acc = reinterpret_cast<float*>(smem + kE2SmemAcc);
        for (long long unit = u0; unit < u1; ++unit) {
            for (int j = 0; j < a.k; ++j) {
                e2_build_h1<true>(a, s1, t1, unit, j, A, hpos, ht);
                for (int half = 0; half < 2; ++half) {
                    e2_mma(d, A, base + kE2SmemF + (uint32_t)half * kE2Block, 0u);
#pragma unroll
                    for (int i = 0; i < 32; ++i) d[i] += b2[64 * half + e2_col(i >> 2) + (i & 1)];
                    e2_dy2(a, v2, unit, j, half, d);
                    uint32_t ovf = 0u;
#pragma unroll
                    for (int i = 0; i < 32; i += 2) {
                        const int r = e2_row((i >> 1) & 1), c = 64 * half + e2_col(i >> 2);
                        uint32_t pc[3];
                        split_pair<3>(d[i], d[i + 1], pc, ovf);
#pragma unroll
                        for (int pi = 0; pi < 3; ++pi) {
                            *reinterpret_cast<uint16_t*>(dyt + pi * 2 * kE2Piece + swz_off_bf16(c, r, kE2C2)) = (uint16_t)(pc[pi] & 0xffffu);
                            *reinterpret_cast<uint16_t*>(dyt + pi * 2 * kE2Piece + swz_off_bf16(c + 1, r, kE2C2)) = (uint16_t)(pc[pi] >> 16);
                        }
                    }
                }
                fence_proxy_async_smem();
                __syncthreads();
                // dW2[c1][c2] of this block = h1^T (M = C1, K = 64 edges) . dy2 (N = C2): both operands from shared memory
                float dw[2][32];
                wg_fence();
#pragma unroll
                for (int tt = 0; tt < Split<3>::kTerms; ++tt)
#pragma unroll
                    for (int s = 0; s < 4; ++s)
#pragma unroll
                        for (int nh = 0; nh < 2; ++nh)
                            wg_mma_ss_bf16(dw[nh], wg_desc(base + kE2SmemHt + Split<3>::a(tt) * kE2Piece + (uint32_t)s * 32u),
                                           wg_desc(base + kE2SmemDyt + Split<3>::w(tt) * 2u * kE2Piece + (uint32_t)nh * 8192u + (uint32_t)s * 32u),
                                           (tt | s) ? 1u : 0u);
                wg_commit();
                wg_wait_all();
                wg_fence_acc(dw[0]);
                wg_fence_acc(dw[1]);
                // each thread adds its own fragment positions: no two threads touch one accumulator
#pragma unroll
                for (int nh = 0; nh < 2; ++nh)
#pragma unroll
                    for (int i = 0; i < 32; ++i)
                        acc[e2_row((i >> 1) & 1) * kE2C2 + 64 * nh + e2_col(i >> 2) + (i & 1)] += dw[nh][i];
                __syncthreads();         // the next block overwrites the staged pieces
            }
        }
        for (int i = tid; i < kE2C1 * kE2C2; i += kE2Threads) a.part[(size_t)chunk * kE2C1 * kE2C2 + i] = acc[i];
    } else {
        for (long long unit = u0; unit < u1; ++unit) {
            for (int j = 0; j < a.k; ++j) {
                float dh[32];
                for (int half = 0; half < 2; ++half) {
                    e2_build_h1<false>(a, s1, t1, unit, j, A, hpos, nullptr);      // rebuilt per half: A is not live across the dh1 product
                    e2_mma(d, A, base + kE2SmemF + (uint32_t)half * kE2Block, 0u);
#pragma unroll
                    for (int i = 0; i < 32; ++i) d[i] += b2[64 * half + e2_col(i >> 2) + (i & 1)];
                    e2_dy2(a, v2, unit, j, half, d);
                    uint32_t D[3][4][4], ovf = 0u;
#pragma unroll
                    for (int i = 0; i < 32; i += 2) {
                        uint32_t pc[3];
                        split_pair<3>(d[i], d[i + 1], pc, ovf);
#pragma unroll
                        for (int pi = 0; pi < 3; ++pi) D[pi][i >> 3][((i >> 2) & 1) << 1 | ((i >> 1) & 1)] = pc[pi];
                    }
                    e2_mma(dh, D, base + kE2SmemX + (uint32_t)half * kE2Block, (uint32_t)half);
                }
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const long long p = unit * kE2Rows + e2_row(hr);
                    if (p >= a.points) continue;
#pragma unroll
                    for (int jb = 0; jb < 8; ++jb) {
                        const int i = 4 * jb + 2 * hr;
                        *reinterpret_cast<float2*>(a.dz1 + ((size_t)p * a.k + j) * kE2C1 + e2_col(jb)) =
                            make_float2((hpos >> i) & 1u ? dh[i] : 0.f, (hpos >> (i + 1)) & 1u ? dh[i + 1] : 0.f);
                    }
                }
            }
        }
    }
}

// layer 2's batch-norm sums are point-sized: the masked edges of a positive maximum all carry dz2 = R, and share the winning value.
// One thread per channel walks the 64 centres of a unit in order: partial[unit] = [sum dz2 | sum dz2 * xhat2].  partial == NULL (frozen
// batch norm): R only, ywin and mean_inv are not read.
__global__ void __launch_bounds__(kE2C2) edge2_bn2_sums_kernel(long long points, const float* __restrict__ pooled, const uint32_t* __restrict__ mask,
                                                               const float* __restrict__ ywin, const float* __restrict__ mean_inv,
                                                               const float* __restrict__ dout, float* __restrict__ R, float* __restrict__ partial) {
    const int c = threadIdx.x;
    const bool sums = partial != nullptr;
    const float mu = sums ? __ldg(mean_inv + c) : 0.f, inv = sums ? __ldg(mean_inv + kE2C2 + c) : 0.f;
    float sb = 0.f, sg = 0.f;
    for (long long p = (long long)blockIdx.x * kE2Rows; p < points && p < ((long long)blockIdx.x + 1) * kE2Rows; ++p) {
        const size_t o = (size_t)p * kE2C2 + c;
        const float cnt = (float)__popc(__ldg(mask + o));
        const float r = __ldg(pooled + o) > 0.f ? __fdiv_rn(__ldg(dout + o), cnt) : 0.f;
        R[o] = r;
        if (!sums) continue;
        sb = fmaf(r, cnt, sb);
        sg = fmaf(r * cnt, (__ldg(ywin + o) - mu) * inv, sg);
    }
    if (!sums) return;
    partial[(size_t)blockIdx.x * 2 * kE2C2 + c] = sb;
    partial[(size_t)blockIdx.x * 2 * kE2C2 + kE2C2 + c] = sg;
}

// layer 1's batch-norm sums from dz1: 4 x 64 threads, thread (q, c) walks centres q, q + 4, .. of the unit; the four are added in order
__global__ void __launch_bounds__(4 * kE2C1) edge2_bn1_sums_kernel(long long points, int n, int k, const float* __restrict__ PQ,
                                                                   const int* __restrict__ nn, const float* __restrict__ mean_inv,
                                                                   const float* __restrict__ dz1, float* __restrict__ partial) {
    __shared__ float red[4][2][kE2C1];
    const int c = threadIdx.x & (kE2C1 - 1), q = threadIdx.x / kE2C1;
    const float mu = __ldg(mean_inv + c), inv = __ldg(mean_inv + kE2C1 + c);
    float sb = 0.f, sg = 0.f;
    for (int r = q; r < kE2Rows; r += 4) {
        const long long p = (long long)blockIdx.x * kE2Rows + r;
        if (p >= points) break;
        const long long base = (p / n) * n;
        const float qv = __ldg(PQ + (size_t)p * 2 * kE2C1 + c);
        for (int j = 0; j < k; ++j) {
            const int nb = __ldg(nn + (size_t)p * k + j);
            const float y = __fadd_rn(qv, __ldg(PQ + (size_t)(base + nb) * 2 * kE2C1 + kE2C1 + c));
            const float dz = __ldg(dz1 + ((size_t)p * k + j) * kE2C1 + c);
            sb += dz;
            sg = fmaf(dz, (y - mu) * inv, sg);
        }
    }
    red[q][0][c] = sb;
    red[q][1][c] = sg;
    __syncthreads();
    if (q < 2) {
        const float s = red[0][q][c] + red[1][q][c] + red[2][q][c] + red[3][q][c];
        partial[(size_t)blockIdx.x * 2 * kE2C1 + q * kE2C1 + c] = s;
    }
}

size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
long long e2_units(long long points) { return (points + kE2Rows - 1) / kE2Rows; }
long long e2_chunks(long long points) { return (e2_units(points) + kE2Chunk - 1) / kE2Chunk; }

// workspace (every segment 256-byte aligned):
//   imgF, imgX, coef1, coef2, part1 (units, 2, C1), part2 (max(units, chunks), 2, C2), dz1 (E, C1), then
//   either R (points, C2) + dW2 partials (chunks, C1, C2)   (forward 2 .. backward dh1)
//   or the layer-1 tail (edge_layer_tail)                    (backward, after dz1)
// The layer-1 forward call (psa_edgeconv_train_fwd) uses the same workspace from offset 0.
struct E2Layout {
    size_t imgF, imgX, coef1, coef2, part1, part2, dz1, r, dw2, tail, total;
    E2Layout(int b, int n, int c, int k) {
        const long long points = (long long)b * n, units = e2_units(points);
        imgF = 0;
        imgX = imgF + al256(kE2Image);
        coef1 = imgX + al256(kE2Image);
        coef2 = coef1 + al256(3 * kE2C1 * sizeof(float));
        part1 = coef2 + al256(3 * kE2C2 * sizeof(float));
        part2 = part1 + al256((size_t)units * 2 * kE2C1 * sizeof(float));
        dz1 = part2 + al256((size_t)units * 2 * kE2C2 * sizeof(float));
        r = dz1 + al256((size_t)points * k * kE2C1 * sizeof(float));
        dw2 = r + al256((size_t)points * kE2C2 * sizeof(float));
        const size_t a = dw2 + al256((size_t)e2_chunks(points) * kE2C1 * kE2C2 * sizeof(float));
        tail = r;
        const size_t t = tail + edge_tail_workspace_bytes(b, n, c, k, kE2C1);
        total = a > t ? a : t;
        const size_t l1 = psa_edgeconv_train_workspace_bytes(b, n, c, k, kE2C1);
        if (l1 > total) total = l1;
    }
};

int e2_check(const char* who, int b, int n, int c, int k, int C1, int C2) {
    PSA_REQUIRE(b >= 1 && n >= 1 && c >= 1 && k >= 1 && C1 >= 1 && C2 >= 1, "%s: bad dims b=%d n=%d c=%d k=%d C1=%d C2=%d", who, b, n, c, k, C1, C2);
    PSA_SUPPORTED(C1 == kE2C1 && C2 == kE2C2, "%s: widths C1=%d C2=%d; the two-layer EdgeConv is written for C1=%d, C2=%d", who, C1, C2, kE2C1, kE2C2);
    PSA_SUPPORTED(k <= kE2MaxK, "%s: k=%d neighbours exceed %d (one 32-bit mask word per centre and channel)", who, k, kE2MaxK);
    PSA_SUPPORTED((long long)n * k <= INT_MAX, "%s: n*k = %lld edges per cloud exceed int32", who, (long long)n * k);
    return PSA_OK;
}

int e2_check_ws(const char* who, const void* ws, size_t ws_bytes, size_t need) {
    PSA_REQUIRE(ws != nullptr && ws_bytes >= need, "%s: workspace of %zu bytes required (got %zu)", who, need, ws_bytes);
    PSA_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "%s: workspace must be 256-byte aligned", who);
    return PSA_OK;
}

template <int MODE>
int e2_launch(const E2Args& a, cudaStream_t st) {
    const uint32_t smem = e2_smem_bytes(MODE);
    PSA_CUDA(cudaFuncSetAttribute(edge2_train_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    edge2_train_kernel<MODE><<<(unsigned)((a.units + kE2Chunk - 1) / kE2Chunk), kE2Threads, smem, st>>>(a);
    return check_launch("edge2_train_kernel");
}

int e2_images(const float* W2, uint8_t* ws, const E2Layout& L, bool transposed, cudaStream_t st) {
    edge2_image_kernel<<<32, 256, 0, st>>>(kE2C1, kE2C2, kE2C2, 1, W2, ws + L.imgF);            // B[n = c2][k = c1] = W2[c1][c2]
    int rc = check_launch("edge2_image_kernel");
    if (rc != PSA_OK || !transposed) return rc;
    edge2_image_kernel<<<32, 256, 0, st>>>(kE2C2, kE2C1, 1, kE2C2, W2, ws + L.imgX);            // B[n = c1][k = c2] = W2[c1][c2]
    return check_launch("edge2_image_kernel");
}

E2Args e2_args(int b, int n, int k, const int* nn_idx, const float* PQ, const float* s1, const float* t1, const float* bias2, uint8_t* ws,
               const E2Layout& L) {
    E2Args a = {};
    a.points = (long long)b * n;
    a.units = e2_units(a.points);
    a.n = n; a.k = k;
    a.PQ = PQ; a.nn = nn_idx; a.s1 = s1; a.t1 = t1; a.b2 = bias2;
    a.imgF = ws + L.imgF; a.imgX = ws + L.imgX;
    return a;
}

}  // namespace
}  // namespace psa

using namespace psa;

extern "C" size_t psa_edgeconv2_train_workspace_bytes(int b, int n, int c, int k, int C1, int C2) {
    if (b < 1 || n < 1 || c < 1 || k < 1 || k > kE2MaxK || C1 != kE2C1 || C2 != kE2C2 || (long long)n * k > INT_MAX) return 0;
    return E2Layout(b, n, c, k).total;
}

extern "C" int psa_edgeconv2_train_fwd(int b, int n, int c, int k, int C1, int C2, const int* nn_idx, const float* PQ, const float* scale1,
                                       const float* shift1, const float* W2, const float* bias2, float* stats2, void* workspace, size_t workspace_bytes,
                                       psa_stream_t stream) {
    int rc = e2_check("edgeconv2_train_fwd", b, n, c, k, C1, C2);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(nn_idx && PQ && scale1 && shift1 && W2 && stats2, "edgeconv2_train_fwd: null buffer");
    rc = e2_check_ws("edgeconv2_train_fwd", workspace, workspace_bytes, psa_edgeconv2_train_workspace_bytes(b, n, c, k, C1, C2));
    if (rc != PSA_OK) return rc;
    cudaStream_t st = as_stream(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    const E2Layout L(b, n, c, k);
    rc = e2_images(W2, ws, L, false, st);
    if (rc != PSA_OK) return rc;
    E2Args a = e2_args(b, n, k, nn_idx, PQ, scale1, shift1, bias2, ws, L);
    a.part = reinterpret_cast<float*>(ws + L.part2);
    rc = e2_launch<kE2Stats>(a, st);
    if (rc != PSA_OK) return rc;
    return reduce_partials((int)e2_chunks(a.points), 2 * kE2C2, a.part, stats2, st);
}

extern "C" int psa_edgeconv2_train_pool(int b, int n, int c, int k, int C1, int C2, const int* nn_idx, const float* PQ, const float* scale1,
                                        const float* shift1, const float* W2, const float* bias2, const float* scale2, const float* shift2,
                                        float* pooled, unsigned int* mask, float* ywin, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = e2_check("edgeconv2_train_pool", b, n, c, k, C1, C2);
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(nn_idx && PQ && scale1 && shift1 && W2 && scale2 && shift2 && pooled && mask && ywin, "edgeconv2_train_pool: null buffer");
    rc = e2_check_ws("edgeconv2_train_pool", workspace, workspace_bytes, psa_edgeconv2_train_workspace_bytes(b, n, c, k, C1, C2));
    if (rc != PSA_OK) return rc;
    cudaStream_t st = as_stream(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    const E2Layout L(b, n, c, k);
    rc = e2_images(W2, ws, L, false, st);
    if (rc != PSA_OK) return rc;
    E2Args a = e2_args(b, n, k, nn_idx, PQ, scale1, shift1, bias2, ws, L);
    a.s2 = scale2; a.t2 = shift2; a.pooled = pooled; a.mask = mask; a.ywin = ywin;
    return e2_launch<kE2Pool>(a, st);
}

extern "C" int psa_edgeconv2_train_bwd(int b, int n, int c, int k, int C1, int C2, const float* x, const int* nn_idx, const float* W1, const float* PQ,
                                       const float* scale1, const float* shift1, const float* gamma1, const float* mean_inv1, const float* W2,
                                       const float* bias2, const float* gamma2, const float* mean_inv2, const float* pooled, const unsigned int* mask,
                                       const float* ywin, const float* dout, float* dW1, float* dgamma1, float* dbeta1, float* dW2, float* dgamma2,
                                       float* dbeta2, float* dx, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = e2_check("edgeconv2_train_bwd", b, n, c, k, C1, C2);
    if (rc != PSA_OK) return rc;
    PSA_SUPPORTED(n <= kE2MaxCloud, "edgeconv2_train_bwd: n=%d points per cloud exceed %d (reverse neighbour lists)", n, kE2MaxCloud);
    PSA_REQUIRE(x && nn_idx && W1 && PQ && scale1 && shift1 && gamma1 && mean_inv1 && W2 && gamma2 && mean_inv2 && pooled && mask && ywin && dout &&
                dW1 && dgamma1 && dbeta1 && dW2 && dgamma2 && dbeta2 && dx, "edgeconv2_train_bwd: null buffer");
    rc = e2_check_ws("edgeconv2_train_bwd", workspace, workspace_bytes, psa_edgeconv2_train_workspace_bytes(b, n, c, k, C1, C2));
    if (rc != PSA_OK) return rc;
    cudaStream_t st = as_stream(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    const E2Layout L(b, n, c, k);
    const long long points = (long long)b * n, units = e2_units(points), edges = points * k;
    float* coef1 = reinterpret_cast<float*>(ws + L.coef1);
    float* coef2 = reinterpret_cast<float*>(ws + L.coef2);
    float* part1 = reinterpret_cast<float*>(ws + L.part1);
    float* part2 = reinterpret_cast<float*>(ws + L.part2);
    float* dz1 = reinterpret_cast<float*>(ws + L.dz1);
    float* R = reinterpret_cast<float*>(ws + L.r);
    float* pdw = reinterpret_cast<float*>(ws + L.dw2);
    rc = e2_images(W2, ws, L, true, st);
    if (rc != PSA_OK) return rc;
    // layer 2: batch-norm sums -> dgamma2, dbeta2, ca2, cb2, cc2
    edge2_bn2_sums_kernel<<<(unsigned)units, kE2C2, 0, st>>>(points, pooled, mask, ywin, mean_inv2, dout, R, part2);
    rc = check_launch("edge2_bn2_sums_kernel");
    if (rc != PSA_OK) return rc;
    rc = launch_bn_bwd_final((int)units, kE2C2, edges, part2, gamma2, mean_inv2, dgamma2, dbeta2, coef2, coef2 + kE2C2, coef2 + 2 * kE2C2, st);
    if (rc != PSA_OK) return rc;
    E2Args a = e2_args(b, n, k, nn_idx, PQ, scale1, shift1, bias2, ws, L);
    a.mask = const_cast<uint32_t*>(mask); a.R = R; a.coef2 = coef2;
    // dW2 = sum_e h1^T dy2
    a.part = pdw;
    rc = e2_launch<kE2Dw2>(a, st);
    if (rc != PSA_OK) return rc;
    rc = reduce_partials((int)e2_chunks(points), kE2C1 * kE2C2, pdw, dW2, st);
    if (rc != PSA_OK) return rc;
    // dz1 = (dy2 . W2^T) [h1 > 0]
    a.dz1 = dz1;
    rc = e2_launch<kE2Dh1>(a, st);
    if (rc != PSA_OK) return rc;
    // layer 1: batch-norm sums -> dgamma1, dbeta1, ca1, cb1, cc1, then dQ, dP and the dense tail (R and the dW2 partials are dead here)
    edge2_bn1_sums_kernel<<<(unsigned)units, 4 * kE2C1, 0, st>>>(points, n, k, PQ, nn_idx, mean_inv1, dz1, part1);
    rc = check_launch("edge2_bn1_sums_kernel");
    if (rc != PSA_OK) return rc;
    rc = launch_bn_bwd_final((int)units, kE2C1, edges, part1, gamma1, mean_inv1, dgamma1, dbeta1, coef1, coef1 + kE2C1, coef1 + 2 * kE2C1, st);
    if (rc != PSA_OK) return rc;
    return edge_layer_tail(b, n, c, k, kE2C1, x, nn_idx, W1, PQ, scale1, shift1, coef1, nullptr, nullptr, dz1, dW1, dx, ws + L.tail, st);
}

extern "C" int psa_edgeconv2_frozen_bwd(int b, int n, int c, int k, int C1, int C2, const float* x, const int* nn_idx, const float* W1,
                                        const float* PQ, const float* scale1, const float* shift1, const float* W2, const float* bias2,
                                        const float* scale2, const float* pooled, const unsigned int* mask, const float* ywin, const float* dout,
                                        float* dx, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = e2_check("edgeconv2_frozen_bwd", b, n, c, k, C1, C2);
    if (rc != PSA_OK) return rc;
    PSA_SUPPORTED(n <= kE2MaxCloud, "edgeconv2_frozen_bwd: n=%d points per cloud exceed %d (reverse neighbour lists)", n, kE2MaxCloud);
    PSA_REQUIRE(x && nn_idx && W1 && PQ && scale1 && shift1 && W2 && scale2 && pooled && mask && ywin && dout && dx,
                "edgeconv2_frozen_bwd: null buffer");
    rc = e2_check_ws("edgeconv2_frozen_bwd", workspace, workspace_bytes, psa_edgeconv2_train_workspace_bytes(b, n, c, k, C1, C2));
    if (rc != PSA_OK) return rc;
    cudaStream_t st = as_stream(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    const E2Layout L(b, n, c, k);
    const long long points = (long long)b * n, units = e2_units(points);
    float* coef1 = reinterpret_cast<float*>(ws + L.coef1);
    float* coef2 = reinterpret_cast<float*>(ws + L.coef2);
    float* dz1 = reinterpret_cast<float*>(ws + L.dz1);
    float* R = reinterpret_cast<float*>(ws + L.r);
    rc = e2_images(W2, ws, L, true, st);
    if (rc != PSA_OK) return rc;
    // layer 2: the max's gradient routed to the masked edges (no batch-norm sums), dy2 = scale2 * dz2
    edge2_bn2_sums_kernel<<<(unsigned)units, kE2C2, 0, st>>>(points, pooled, mask, ywin, nullptr, dout, R, nullptr);
    rc = check_launch("edge2_bn2_sums_kernel");
    if (rc != PSA_OK) return rc;
    rc = frozen_coef(kE2C2, scale2, coef2, st);
    if (rc != PSA_OK) return rc;
    // dz1 = (dy2 . W2^T) [h1 > 0]
    E2Args a = e2_args(b, n, k, nn_idx, PQ, scale1, shift1, bias2, ws, L);
    a.mask = const_cast<uint32_t*>(mask); a.R = R; a.coef2 = coef2; a.dz1 = dz1;
    rc = e2_launch<kE2Dh1>(a, st);
    if (rc != PSA_OK) return rc;
    // layer 1: dy1 = scale1 * dz1, then dQ, dP and dx (R is dead here)
    rc = frozen_coef(kE2C1, scale1, coef1, st);
    if (rc != PSA_OK) return rc;
    return edge_layer_tail(b, n, c, k, kE2C1, x, nn_idx, W1, PQ, scale1, shift1, coef1, nullptr, nullptr, dz1, nullptr, dx, ws + L.tail, st);
}
