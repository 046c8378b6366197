// tc_mlp.cu -- the grouped shared MLP of a set-abstraction level and the dense layers on the Hopper tensor cores
// (wgmma, A from registers, B from shared memory), hand-written PTX wrappers in tc_common.cuh.
//
// What the reference does (pointnet2/utils/pointnet_util.py:113-127): group_point -> (B,m,K,3+C) tensor -> three
// cuDNN 1x1 convs over B*m*K rows -> reduce_max.  What the kernels here do per tile (64 or 128 rows):
//
//   layer 1   is never a GEMM over grouped rows.  s ((x_j - c) . Wx + f_j . Wf) + t  =  V[j] - c . (s Wx)   with
//             V = s (points . W1[3:,:] + xyz . W1[:3,:]) + t computed ONCE per source point (K-fold fewer rows, a dense-layer
//             launch); each thread gathers its part of the V rows, subtracts the centre term of its columns (3 FMAs per column
//             and neighbourhood, shared by its rows), applies the ReLU and keeps the result in registers as the A operand of
//             layer 2 -- the (B,m,K,C) tensors of the reference never exist, not even in shared memory.  Levels without
//             input features evaluate t + (x_j - c) . (s Wx) per row.
//   layers 2+ wgmma, A from registers, B = weights in shared memory in the canonical K-major SWIZZLE_128B layout, dropped
//             there by cp.async.bulk from pre-arranged images; D in registers, whose layout is that of the next A operand.
//   max-pool  the last epilogue reduces each neighbourhood's rows in-thread and across the warp with shuffles, folds them into
//             a shared-memory row per neighbourhood with atomicMax, and writes (B,m,C_out) coalesced once per chunk.
//
// Kernels (both templated on NP, the pieces per operand -- Split<NP> in tc_common.cuh):
//   tc_sa_kernel<NP,..>       SA level (specialised on its shape); optional centre weights = multi-layer EdgeConv over 3-D points
//   tc_dense_kernel<NP,NC>    dense layer on the shared ring (ring_gemm.cuh), units of 128 rows x 64 NC channels claimed from a
//                             counter; also the training-mode forward (previous batch norm applied on load, column statistics
//                             in the epilogue)
//   tc_group_all_kernel<..>   a three-layer group-all level with 128 points per cloud, fp16x2: one four-CTA cluster per cloud,
//                             the activations between the layers kept in the cluster's shared memory
// fp32 parity: operands are quantised by this code, so the tensor core only ever sees exactly representable values; fp32
// accumulation in the tensor core truncates, hence small terms first and K cut into <= 128-wide pieces (tests hold 1e-5 vs fp64).
//   NP = 2 (inference default): two fp16 pieces, three MMAs per product, weights scaled per output column by a power of two (see
//           the weight images below); every kernel tracks the leading activation pieces it stores and raises a device-side flag
//           when one leaves the fp16 range or a weight is not finite -- the launchers then rerun the op on the NP = 3
//           instantiation (enqueued unconditionally, a no-op unless the flag is set: `run_if`);
//   NP = 3 (psa_set_mlp_mode(2), the guarded rerun, the training forward): three bf16 pieces, six MMAs per product.
// Levels the SA kernel cannot hold run on the fp32-FMA fused kernel of mlp.cu.
#include <float.h>
#include <stdlib.h>

#include <algorithm>
#include <atomic>
#include <type_traits>

#include "common.cuh"
#include "mlp_internal.cuh"
#include "ring_gemm.cuh"
#include "tc_common.cuh"

namespace psa {

using namespace tc;

constexpr int kMaxTcLayers = 2;

// ------------------------------------------------------------------------------------------------------------------
// Weight images.  A tensor layer W (K x N, row-major, fp32) is pre-arranged once per weight set (tc_prep_weights_kernel) into
// blocks that can be dropped into shared memory by a single cp.async.bulk and fed to wgmma unchanged:
//   block (nt, kc) covers output channels [nt*Nt, nt*Nt+Nt) x input channels [kc*64, kc*64+64): NP 16-bit pieces
//   (every piece exactly representable), each [Nt][64] K-major SWIZZLE_128B, Nt*128 B per piece; blocks stored in (nt major,
//   kc minor) order.  2 NP bytes per weight.
//   fp16x2 images hold column n of W times 2^e_n, with e_n chosen so that the column's largest |w| lands in [2^10, 2^11)
//   (tc_col_scale_kernel): the two fp16 pieces then keep 22 bits relative to that weight whatever the scale of the weights.
//   Unscaled, a weight below 0.125 has a subnormal second piece and keeps only an absolute 2^-25, which batch norm calibrated
//   to small weights multiplies by up to 31.6 gamma.  The image carries 2^-e_n per column; the kernels fold it into the scale
//   of their epilogue, and bring what they add to the accumulators before it into the same units (exact: powers of two).
// ------------------------------------------------------------------------------------------------------------------
// (the byte layout helpers tc_block_bytes .. tc_image_alloc_bytes are in tc_common.cuh, shared with spider.cu)

struct TcArgs {
    long long groups;      // neighbourhoods = b*m
    int K;                 // rows per neighbourhood (32 | 64 | 128)
    int n, m;              // dataset points / queries per cloud
    const float* xyz;      // (b,n,3)
    const float* new_xyz;  // (b,m,3)
    const float* uf;       // (b*n, C1) = V = s (points . W1[3:,:] + xyz . W1[:3,:]) + t, or null when the level has no input features
    const int* idx;        // (groups, K)
    float* out;            // (groups, Ntot[last])
    // layer 1 (FMA path)
    const float* w1c;      // optional (3, C1): weights applied to the CENTRE coordinates new_xyz (EdgeConv's x_i part), or null
    const float* w1x;      // (3, C1): rows 0..2 of W1
    const float* s1;       // scale or null
    const float* t1;       // shift
    int C1, relu1;
    // tensor layers
    int nl;
    const uint8_t* image[kMaxTcLayers];   // weight images (global)
    const float* s[kMaxTcLayers];
    const float* t[kMaxTcLayers];
    int relu[kMaxTcLayers];
    int Kd[kMaxTcLayers], Ntot[kMaxTcLayers];
    int stream_last;       // 1: the last layer's weights do not fit next to the others -> one 64-channel chunk at a time
    int joint;             // tc_sa_kernel: both warpgroups on one 128-row pass, every row computed (set by the launcher)
    unsigned int* tile_counter;   // zeroed before the launch: tiles are handed out dynamically (CTAs that start late or
                                  // share their SM with another stream's kernels simply take fewer)
    int np;                       // operand pieces: 2 (fp16x2) or 3 (bf16x3)
    unsigned int* ovf;            // np = 2: set to 1 when an activation left the fp16 range or a weight is not finite (the result is then invalid)
    const unsigned int* run_if;   // non-null: the launch is a no-op unless *run_if != 0 (the np = 3 rerun of a flagged launch)
    const unsigned int* wflag[kMaxTcLayers];     // np = 2: trailer word of each weight image
    const float* colscale[kMaxTcLayers];         // np = 2: column factors 2^-e_n of each weight image (folded into the layer's scale)
};

// ------------------------------------------------------------------------------------------------------------------
// Fragment helpers of the warpgroup kernels (layout in tc_common.cuh).  A 128-row tile is two warpgroups; warp w of the
// CTA holds tile rows 16w + g and 16w + g + 8 (g = lane / 4, t = lane % 4).
// ------------------------------------------------------------------------------------------------------------------
// split the pair (x0, x1) of consecutive k into NP pieces and store piece i as register r of K step s of A
template <int NP, int S>
__device__ __forceinline__ void put_a(uint32_t (&A)[NP][S][4], int s, int r, float x0, float x1, uint32_t& ovf) {
    uint32_t p[NP];
    split_pair<NP>(x0, x1, p, ovf);
#pragma unroll
    for (int i = 0; i < NP; ++i) A[i][s][r] = p[i];
}

// max over the 16 rows of a warp of columns (8j + 2t, 8j + 2t + 1): in-thread over rows g / g + 8, then across g
__device__ __forceinline__ float warp_rowmax16(float lo, float hi) {
    float m = fmaxf(lo, hi);
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
    return m;
}
// the same max, reduce-scattered over a whole 64-column chunk: with v[2j + e] = this thread's max over rows g, g + 8 of column
// 8j + 2t + e, each step across lane bit 4, 3, 2 (= bit 2, 1, 0 of g) keeps the half of the columns whose j has that bit of g,
// 8 + 4 + 2 shuffles, and lane (g, t) ends with the 16-row max of columns 8g + 2t, 8g + 2t + 1.  One step: keep v[0..H) or
// v[H..2H) by `up`, the partner across lane bit 2H keeps the other half (the caller does the first step as it forms v, so
// that only half of the 16 values are live at once).
template <int H, int S>
__device__ __forceinline__ void colmax_halve(float (&v)[S], bool up) {
#pragma unroll
    for (int i = 0; i < H; ++i) {
        const float lo = v[i], hi = v[H + i];
        v[i] = fmaxf(up ? hi : lo, __shfl_xor_sync(0xffffffffu, up ? lo : hi, 2 * H));
    }
}
__device__ __forceinline__ float warp_rowsum16(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    return v;
}

// fp16x2 images: the column factor 2^-e_n of every column of W (K x N) into colscale.  Block (32, 8): 32 columns, the rows strided
// over 8 threads.  A column holding a non-finite weight keeps e_n = 0 and sets the trailer word (the op is then rerun with bf16x3
// operands, which give what fp32 gives); finite weights scaled this way cannot leave the fp16 range.  e_n <= 64 keeps 2^-e_n and
// the scales it is folded into normal (columns of weights below 2^-54 are scaled by 2^64 only).
__global__ void __launch_bounds__(256) tc_col_scale_kernel(int K, int N, const float* __restrict__ W, float* __restrict__ colscale,
                                                           unsigned int* __restrict__ trailer) {
    __shared__ float s_max[8][32];
    __shared__ int s_bad[8][32];
    const int n = blockIdx.x * 32 + threadIdx.x;
    float m = 0.f;
    bool bad = false;
    if (n < N)
        for (int k = threadIdx.y; k < K; k += 8) {
            const float w = __ldg(W + (size_t)k * N + n);
            bad = bad || !isfinite(w);
            m = fmaxf(m, fabsf(w));
        }
    s_max[threadIdx.y][threadIdx.x] = m;
    s_bad[threadIdx.y][threadIdx.x] = bad;
    __syncthreads();
    if (threadIdx.y != 0 || n >= N) return;
    for (int y = 1; y < 8; ++y) { m = fmaxf(m, s_max[y][threadIdx.x]); bad = bad || s_bad[y][threadIdx.x]; }
    int e = 0;
    if (!bad && m > 0.f) e = min(137 - (int)(__float_as_uint(m) >> 23), 64);   // m in [2^(E-127), 2^(E-126)): m 2^e in [2^10, 2^11)
    colscale[n] = __int_as_float((127 - e) << 23);
    if (bad) atomicOr(trailer, 1u);
}

// colscale: fp16x2, the column factors of tc_col_scale_kernel (the weights are stored divided by them, exactly); bf16x3: null
template <int NP>
__global__ void tc_prep_weights_kernel(int K, int Kp, int N, int Nt, const float* __restrict__ W, const float* __restrict__ colscale,
                                       uint8_t* __restrict__ image, const unsigned int* __restrict__ run_if) {
    if (run_if != nullptr && *run_if == 0u) return;
    const int KC = Kp / 64;
    const uint32_t bb = tc_block_bytes(Nt, NP), piece = (uint32_t)Nt * 128u;
    uint32_t unused = 0u;                  // split_pair's range tracking: scaled finite weights stay inside the fp16 range
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < Kp * N; e += gridDim.x * blockDim.x) {
        const int n = e % N, k = e / N;
        float w = k < K ? __ldg(W + e) : 0.f;
        if (NP == 2) w *= pow2_rcp(__ldg(colscale + n));
        uint32_t pc[NP];
        split_pair<NP>(w, 0.f, pc, unused);
        uint8_t* blk = image + (size_t)((n / Nt) * KC + (k >> 6)) * bb;
        const uint32_t off = swz_off_bf16(n % Nt, k & 63, Nt);
#pragma unroll
        for (int i = 0; i < NP; ++i) *reinterpret_cast<uint16_t*>(blk + i * piece + off) = (uint16_t)(pc[i] & 0xffffu);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// tc_sa_kernel -- one set-abstraction level (e.g. PointNet++ SA2: 131 -> 128 -> 128 -> 256 over 64-point neighbourhoods).
//   CTA = 256 threads = two warpgroups, persistent (as many per SM as fit), chunks of neighbourhoods claimed dynamically (a CTA
//   that starts late or shares its SM with another stream simply takes fewer).  K <= 64: each warpgroup works on its own
//   64-row passes, out of step with the other, so one's gathers and FMA epilogues overlap the other's wgmma, and computes only
//   the rows of each neighbourhood before its ball-query padding (16-row slots packed back to back); K = 128 or a streamed
//   last layer: the two work together on 128-row passes of whole neighbourhoods.  NL = 2: layer 1's gathers are issued one
//   pass ahead.
//   * layer 1 on the FMA pipe: each thread evaluates V[j] + c . s (Wc - Wx) (levels with input features) or
//     t + (x_j - c) . s Wx (+ c . s Wc), and the ReLU for the rows and channels of ITS A fragment and splits the result into
//     NP pieces -- straight into registers;
//   * inner tensor layers: wgmma with A from registers, B = weight image in shared memory; the D fragment goes through
//     affine + ReLU + split and is the next layer's A fragment (same register layout), nothing is staged;
//   * last layer in 64-channel chunks: wgmma, affine + ReLU, max over each neighbourhood's rows (in-thread, shuffles across
//     the warp, shared atomicMax across warps and passes), coalesced (B,m,C_out) stores at the end of each chunk of
//     neighbourhoods.
//   Weights of every layer are resident in shared memory (one TMA bulk load per CTA); a last layer that does not fit next to
//   the others is streamed one 64-channel chunk at a time through a two-slot ring, one chunk ahead.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kSaNt = 64;                        // tile width of the SA weight images
constexpr int kSaThreads = 256;
constexpr uint32_t kSmemBudget = 220u * 1024u;   // dynamic shared memory (incl. 1 KB alignment) next to the static arrays

struct TcSaLayout {
    uint32_t w[kMaxTcLayers];    // resident layers
    uint32_t ring[2];            // streamed last layer: one 64-channel chunk per slot
    uint32_t ring_bytes;
    uint32_t vec, total;
};

__host__ __device__ inline TcSaLayout tc_sa_layout(const TcArgs& a) {
    TcSaLayout L;
    uint32_t off = 0;
#pragma unroll
    for (int l = 0; l < kMaxTcLayers; ++l) {      // constant indices: the layout stays in registers inside the kernel
        L.w[l] = off;
        if (l < a.nl && !(a.stream_last && l == a.nl - 1)) off += (uint32_t)tc_image_bytes(a.Kd[l], a.Ntot[l], a.np);
    }
    L.ring_bytes = a.stream_last ? (uint32_t)(a.Kd[a.nl - 1] / 64) * tc_block_bytes(kSaNt, a.np) : 0u;
    L.ring[0] = off; off += L.ring_bytes;
    L.ring[1] = off; off += L.ring_bytes;
    L.vec = off;
    off += 7u * a.C1 * 4u;       // w1x (3 C1), w1c (3 C1), t1
#pragma unroll
    for (int l = 0; l < kMaxTcLayers; ++l) off += l < a.nl ? 2u * a.Ntot[l] * 4u : 0u;
    L.total = off;
    return L;
}

// neighbourhoods per chunk, the work a unit of tc_sa_kernel claims at a time: one 128-row pass for a joint unit (K = 128 or a
// streamed last layer), 512 rows before padding is skipped for a warpgroup unit -- few enough chunks per unit stay that the
// end of the grid is balanced (PointNet++ SA2: 512 chunks for 264 units), enough neighbourhoods per chunk that its last pass
// is mostly full
__host__ __device__ inline int sa_chunk(int K, bool joint) { return (joint ? 128 : 512) / K; }
// columns of a unit's pooling buffer: every column of the last layer, or the 64 of the ring slot being consumed when it streams
__host__ __device__ inline int sa_pool_cols(const TcArgs& a) { return a.stream_last ? 64 : a.Ntot[a.nl - 1]; }
// shared memory of the pooling buffers, after the layout: per unit, one row of sa_pool_cols words per neighbourhood of its chunk
__host__ __device__ inline uint32_t sa_pool_bytes(const TcArgs& a) {
    return (a.joint ? 1u : 2u) * (uint32_t)sa_chunk(a.K, a.joint) * (uint32_t)sa_pool_cols(a) * 4u;
}
// a float as an int that orders like it (shared atomicMax has no float form): the bits of a value >= +0, the magnitude bits
// flipped below it.  The map is its own inverse; -inf maps to kSaPoolEmpty, below every finite value.
__device__ __forceinline__ int sa_pool_code(float x) {
    const int b = __float_as_int(x);
    return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float sa_pool_value(int c) { return __int_as_float(c >= 0 ? c : c ^ 0x7fffffff); }
__device__ __forceinline__ void red_smem_max(uint32_t addr, int v) { asm volatile("red.shared.max.s32 [%0], %1;\n" ::"r"(addr), "r"(v) : "memory"); }
constexpr int kSaPoolEmpty = (int)0x807fffff;

// thread 0: use q of the streamed last layer's ring = 64-channel chunk q % ncl into slot q & 1
__device__ __forceinline__ void sa_fill_ring(uint32_t q, const uint8_t* image, int ncl, const TcSaLayout& L, uint8_t* base, uint64_t* bars) {
    uint64_t* bar = &bars[q & 1];
    mbar_expect_tx(bar, L.ring_bytes);
    const uint8_t* src = image + (size_t)(q % (uint32_t)ncl) * L.ring_bytes;
    for (uint32_t o = 0; o < L.ring_bytes; o += 32768u) bulk_g2s(base + L.ring[q & 1] + o, src + o, min(32768u, L.ring_bytes - o), bar);
}

// D[64 x 64 NCH] (+)= A . W over KS steps of 16 input channels, all piece pairs of Split<NP>: straight-line wgmma (no predicated
// issue, so ptxas keeps the whole sequence asynchronous).  Output chunk c reads the weight blocks at wb + c * cstride.
// sa_mma_issue commits the group and returns with it in flight; sa_mma waits for it.
template <int NP, int KS, int NCH>
__device__ __forceinline__ void sa_mma_issue(float (&d)[NCH][32], const uint32_t (&A)[NP][8][4], uint32_t wb, uint32_t cstride) {
    constexpr uint32_t bb = tc_block_bytes(kSaNt, NP), piece = kSaNt * 128u;
    wg_fence();
#pragma unroll
    for (int tt = 0; tt < Split<NP>::kTerms; ++tt)
#pragma unroll
        for (int s = 0; s < KS; ++s)
#pragma unroll
            for (int c = 0; c < NCH; ++c)
                wg_mma_rs<NP>(d[c], A[Split<NP>::a(tt)][s][0], A[Split<NP>::a(tt)][s][1], A[Split<NP>::a(tt)][s][2], A[Split<NP>::a(tt)][s][3],
                              wg_desc(wb + (uint32_t)c * cstride + (uint32_t)(s >> 2) * bb + Split<NP>::w(tt) * piece + (uint32_t)(s & 3) * 32u),
                              (tt | s) ? 1u : 0u);
    wg_commit();
}
template <int NP, int KS, int NCH>
__device__ __forceinline__ void sa_mma(float (&d)[NCH][32], const uint32_t (&A)[NP][8][4], uint32_t wb, uint32_t cstride) {
    sa_mma_issue<NP, KS, NCH>(d, A, wb, cstride);
    wg_wait_all();
#pragma unroll
    for (int c = 0; c < NCH; ++c) wg_fence_acc(d[c]);
}

#ifdef PSA_SA_STAMPS
// Pass timeline (tools/sa_timing.py builds a separate library with -DPSA_SA_STAMPS; libpsa.so has none of this): lane 0 of the
// first warp of each warpgroup of CTA i < kSaStampCtas writes clock64() at phase k of the unit's pass p < kSaStampPasses
// (SaStamp below; chunk nc of the last layer at kSaChunk0 + 3 nc + {issued, retired, epilogue done}; the two barriers of the
// store at the end of a chunk of neighbourhoods only in the passes that end one).  psa_sa_stamps_clear zeroes the table, so
// that a slot a launch did not reach reads 0.
enum SaStamp { kSaTop, kSaInputs, kSaLayer1, kSaL2Issued, kSaL2Retired, kSaL2Epi, kSaEnd1, kSaEnd2, kSaNextA, kSaNextB, kSaChunk0 };
constexpr int kSaStampCtas = 264, kSaStampPasses = 64, kSaStampPhases = kSaChunk0 + 3 * 4;
__device__ long long g_sa_stamps[kSaStampCtas][2][kSaStampPasses][kSaStampPhases];
extern "C" PSA_API int psa_sa_stamps(long long* dst) {
    return cudaMemcpyFromSymbol(dst, g_sa_stamps, sizeof(g_sa_stamps)) == cudaSuccess ? 0 : 1;
}
extern "C" PSA_API int psa_sa_stamps_clear(void) {
    void* p = nullptr;
    if (cudaGetSymbolAddress(&p, g_sa_stamps) != cudaSuccess) return 1;
    return cudaMemset(p, 0, sizeof(g_sa_stamps)) == cudaSuccess ? 0 : 1;
}
#define SA_STAMP(p, k)                                                                                              \
    do {                                                                                                            \
        if ((threadIdx.x & 127) == 0 && blockIdx.x < kSaStampCtas && (p) < kSaStampPasses && (k) < kSaStampPhases) \
            g_sa_stamps[blockIdx.x][threadIdx.x >> 7][(p)][(k)] = clock64();                                        \
    } while (0)
// the stamp after a volatile store of a value computed from the float r, so the load that wrote r has landed
#define SA_STAMP_AFTER(p, k, r)                                                                                     \
    do {                                                                                                            \
        if ((threadIdx.x & 127) == 0 && blockIdx.x < kSaStampCtas && (p) < kSaStampPasses) {                        \
            volatile long long* p_ = &g_sa_stamps[blockIdx.x][threadIdx.x >> 7][(p)][(k)];                          \
            *p_ = (long long)__float_as_uint(__fmul_rn((r), 0.f));                                                  \
            *p_ = clock64();                                                                                        \
        }                                                                                                           \
    } while (0)
#else
#define SA_STAMP(p, k) \
    do {               \
    } while (0)
#define SA_STAMP_AFTER(p, k, r) \
    do {                        \
    } while (0)
#endif

// Specialised on the level shape: C1 = width of layer 1 (64 | 128), NL = tensor layers (1 | 2), N0 = width of the inner tensor
// layer when NL = 2 (64 | 128).  The last layer's width is a runtime multiple of 64.
template <int NP, int C1, int NL, int N0>
__global__ void __launch_bounds__(kSaThreads, NP == 2 && C1 == 64 && (NL == 1 || N0 == 64) ? 2 : 1)   // 64-(64-)x: two CTAs per SM
tc_sa_kernel(const __grid_constant__ TcArgs a) {
    static_assert((C1 == 64 || C1 == 128) && (NL == 1 || (NL == 2 && (N0 == 64 || N0 == 128))), "unsupported level shape");
    constexpr int last = NL - 1;
    constexpr int KSL = (NL == 2 ? N0 : C1) / 16;            // K steps of the last layer
    // a second last-layer accumulator (the next chunk's wgmma run during this one's epilogue) costs 32 registers: the levels
    // whose layers before the last are 64 wide keep one, so that they stay small enough for two CTAs per SM
    constexpr bool kDouble = !(C1 == 64 && (NL == 1 || N0 == 64));
    if (a.run_if != nullptr && *a.run_if == 0u) return;      // np = 3 rerun of a launch that stayed inside the fp16 range: nothing to do
    constexpr uint32_t bb = tc_block_bytes(kSaNt, NP);
    uint32_t ovf = 0u;                                        // np = 2: packed |max| of every leading piece this thread stores,
                                                              // checked once per pass so that it lives only in layers 1..L-1
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_rbar;                 // resident weights landed
    __shared__ __align__(8) uint64_t s_wbar[2];              // ring slot landed
    __shared__ unsigned int s_chunk[2][2];                   // [unit][table]: the chunk whose slot counts are in s_slots
    __shared__ int s_slots[2][2][16];                        // [unit][table]: 16-row slots of each neighbourhood of a chunk

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const TcSaLayout L = tc_sa_layout(a);

    float* vec = reinterpret_cast<float*>(base + L.vec);
    float* w1x = vec;
    float* w1c = vec + 3 * C1;
    float* t1 = vec + 6 * C1;
    float* sl0 = t1 + C1;                                     // scale / shift of tensor layer 0 ..
    float* tl0 = sl0 + a.Ntot[0];
    float* slL = NL == 2 ? tl0 + a.Ntot[0] : sl0;             // .. and of the last one
    float* tlL = slL + a.Ntot[last];
    // the BN scale of layer 1 is folded into its xyz / centre weights: s (d.Wx + c.Wc) + t = t + d.(s Wx) + c.(s Wc).  With
    // input features the xyz part of the neighbour is in V (x_j.Wx, the affine), and w1c holds s (Wc - Wx): V[j] + c.w1c
    for (int i = tid; i < 3 * C1; i += kSaThreads) {
        const float sc = a.s1 ? __ldg(a.s1 + i % C1) : 1.f;
        w1x[i] = __ldg(a.w1x + i) * sc;
        w1c[i] = (a.w1c ? __ldg(a.w1c + i) : 0.f) * sc - (a.uf ? w1x[i] : 0.f);
    }
    for (int i = tid; i < C1; i += kSaThreads) t1[i] = __ldg(a.t1 + i);
    // the column factors of the fp16x2 weight images are folded into the tensor layers' scales
#pragma unroll
    for (int l = 0; l < NL; ++l)
        for (int i = tid; i < a.Ntot[l]; i += kSaThreads) {
            (l == 0 ? sl0 : slL)[i] = (a.s[l] ? __ldg(a.s[l] + i) : 1.f) * (NP == 2 ? __ldg(a.colscale[l] + i) : 1.f);
            (l == 0 ? tl0 : tlL)[i] = __ldg(a.t[l] + i);
        }
    for (uint32_t i = tid; i < sa_pool_bytes(a) / 4u; i += kSaThreads) reinterpret_cast<int*>(base + L.total)[i] = kSaPoolEmpty;
    if (tid == 0) {
        mbar_init(&s_rbar, 1); mbar_init(&s_wbar[0], 1); mbar_init(&s_wbar[1], 1);
        fence_mbar_init();
    }
    __syncthreads();

    const int NCL = a.Ntot[last] / 64;                        // 64-channel chunks of the last layer
    uint32_t resident = 0;
#pragma unroll
    for (int l = 0; l < NL; ++l)
        if (!(a.stream_last && l == last)) resident += (uint32_t)tc_image_bytes(a.Kd[l], a.Ntot[l], NP);
    if (tid == 0) {
        if (resident) {
            mbar_expect_tx(&s_rbar, resident);
#pragma unroll
            for (int l = 0; l < NL; ++l) {
                if (a.stream_last && l == last) continue;
                const uint32_t bytes = (uint32_t)tc_image_bytes(a.Kd[l], a.Ntot[l], NP);
                for (uint32_t o = 0; o < bytes; o += 32768u) bulk_g2s(base + L.w[l] + o, a.image[l] + o, min(32768u, bytes - o), &s_rbar);
            }
        }
        if (a.stream_last) { sa_fill_ring(0, a.image[last], NCL, L, base, s_wbar); sa_fill_ring(1, a.image[last], NCL, L, base, s_wbar); }
    }
    if (resident) mbar_wait(&s_rbar, 0);

    // Work is done by units of threads.  K <= 64: each warpgroup is a unit of its own, so the two run out of step -- one's
    // gathers, FMA layer and epilogue overlap the other's wgmma.  K = 128 (a neighbourhood spans 128 rows) and a streamed last
    // layer (its ring is consumed by the whole CTA in step): both warpgroups form one unit.  Units synchronise on their own
    // named barrier; no CTA-wide barrier is left in the loop.
    //   A unit claims a chunk of C consecutive neighbourhoods at a time and computes it in passes of one 16-row slot per warp.
    // The ball query pads a neighbourhood by repeating its first index, and a max does not change when a row is repeated: a
    // neighbourhood whose entries from L on all equal idx[0] only needs its first L rows, ceil(L / 16) slots.  The slots of a
    // chunk are packed back to back, so a neighbourhood may start in one pass and end in a later one.  Each warp folds its
    // slot's column maxima into its neighbourhood's row of the unit's pooling buffer with atomicMax, whichever pass it is in;
    // only the chunk's end synchronises the unit, to store the rows and reset them.  Warps past the chunk's last slot
    // recompute that slot and fold it in again (a max is idempotent).  Joint units keep every row: a chunk is then one
    // 128-row pass, as before.
    const int K = a.K;
    const bool joint = a.joint;
    const int W = joint ? 8 : 4;                             // warps of the unit = slots per pass
    const int C = sa_chunk(K, joint);                         // neighbourhoods per chunk (<= 16)
    const int unit = joint ? 0 : warp >> 2;
    const int ubar = 1 + unit, uthreads = 32 * W;             // the unit's named barrier
    const int ut = joint ? tid : tid & 127, uw0 = joint ? 0 : 4 * unit;   // thread index in the unit, first warp of the unit
    const int wl = warp - uw0;                                // warp index in the unit
    const unsigned nchunks = (unsigned)((a.groups + C - 1) / C);
    const int PC = sa_pool_cols(a);
    // the unit's pooling buffer [C][PC]: ordered codes (sa_pool_code), kSaPoolEmpty between chunks; an offset from `base`, so
    // that no pointer of its own is held through the pass
    const uint32_t pool = L.total + (uint32_t)(unit * C * PC) * 4u;

    // slot counts of chunk ch into table b, by the whole unit (read after a unit barrier).  L = 1 + the last j with
    // idx[j] != idx[0] (1 when all are equal), from a ballot per 32 entries; a warp covers 128 entries = 4 neighbourhoods of 32
    // or 2 of 64.  Neighbourhoods past the end take no slot.
    auto fill_table = [&](unsigned ch, int b) {
        const long long g0 = (long long)ch * C;
        if (joint) {
            if (ut < C) s_slots[unit][b][ut] = g0 + ut < a.groups ? K / 16 : 0;
            return;
        }
        const long long r0 = g0 * K + wl * 128, rows = a.groups * K;
        int v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = r0 + 32 * q + lane < rows ? __ldg(a.idx + r0 + 32 * q + lane) : 0;
        if (K == 32) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const unsigned d = __ballot_sync(0xffffffffu, v[q] != __shfl_sync(0xffffffffu, v[q], 0));
                const int nb = 4 * wl + q, Ln = d ? 32 - __clz(d) : 1;
                if (lane == 0) s_slots[unit][b][nb] = g0 + nb < a.groups ? (Ln + 15) >> 4 : 0;
            }
        } else {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int f = __shfl_sync(0xffffffffu, v[2 * h], 0);
                const unsigned lo = __ballot_sync(0xffffffffu, v[2 * h] != f), hi = __ballot_sync(0xffffffffu, v[2 * h + 1] != f);
                const int nb = 2 * wl + h, Ln = hi ? 64 - __clz(hi) : lo ? 32 - __clz(lo) : 1;
                if (lane == 0) s_slots[unit][b][nb] = g0 + nb < a.groups ? (Ln + 15) >> 4 : 0;
            }
        }
    };

    // Layer 1's inputs for this thread's two rows are gathered one pass ahead (NL = 2), while the previous pass's last-layer
    // wgmma run: stage A (neighbour index, centre) once the first chunk is issued, stage B (the V row, or the neighbour
    // coordinates of a level without input features) once the last one is.  The next pass's slot table must be filled by
    // then; it is not when the next pass opens a new chunk (its table is filled at the end of the current one), and both
    // stages then follow that chunk-end store.
    // The 64-float V rows of C1 = 128 levels are held in registers (fp16x2: those levels keep one CTA per SM); other levels
    // load them in layer 1, as do the levels that gather at the top of the pass (nothing to hide the loads behind there).
    constexpr bool kAhead = NL == 2;                          // one-tensor-layer levels (EdgeConv) gather at the top of the pass:
                                                              // measured faster there, the pass is too short to hide the loads
    constexpr bool kHoldU = NP == 2 && C1 == 128 && kAhead;
    constexpr int kUH = kHoldU ? C1 / 8 : 1;                  // float2 per row held
    int incl = 0;                                             // slots of the chunk gather_a last read, prefix (lane i: neighbourhoods
                                                              // 0..i); the chunk's total is lane C - 1's, one shuffle away
    int jn[2];
    long long gn = 0;                                         // the neighbourhood of this warp's slot
    float cx = 0.f, cy = 0.f, cz = 0.f, px[2], py[2], pz[2];
    const float* urow[2];
    float2 uh[2][kUH];                                        // kHoldU: the V row, or the neighbour's coordinates of a level
                                                              // without input features (not px .. pz: six registers SA2 lacks)
    // the chunk's slot total, and the neighbourhood (index in the chunk) of this warp's slot in pass p, both from the prefix.
    // Warps past the chunk's last slot take that slot's.
    auto slot_total = [&]() { return __shfl_sync(0xffffffffu, incl, C - 1); };
    auto slot_nb = [&](int p) { return __popc(__ballot_sync(0xffffffffu, incl <= min(p * W + wl, slot_total() - 1)) & ((1u << C) - 1u)); };
    // stage A of pass p of chunk ch (slot table b)
    auto gather_a = [&](unsigned ch, int b, int p) {
        if (p == 0) {                                         // a new chunk: prefix of its slot table
            incl = lane < C ? s_slots[unit][b][lane] : 0;
#pragma unroll
            for (int o = 1; o < 16; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
            }
        }
        const int ss = min(p * W + wl, slot_total() - 1), nb = slot_nb(p);
        const int start = nb ? __shfl_sync(0xffffffffu, incl, nb - 1) : 0;
        gn = (long long)ch * C + nb;
        const int row = 16 * (ss - start) + g;
#pragma unroll
        for (int i = 0; i < 2; ++i) jn[i] = __ldg(a.idx + gn * K + row + 8 * i);
        const float* c = a.new_xyz + (size_t)gn * 3;
        cx = __ldg(c); cy = __ldg(c + 1); cz = __ldg(c + 2);
    };
    auto gather_b = [&]() {
        const long long bi = gn / a.m;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (a.uf == nullptr) {                            // with input features the neighbour's coordinates are in V
                const float* p = a.xyz + ((size_t)bi * a.n + jn[i]) * 3;
                if constexpr (kHoldU) { uh[i][0] = make_float2(__ldg(p), __ldg(p + 1)); uh[i][1].x = __ldg(p + 2); }
                else { px[i] = __ldg(p); py[i] = __ldg(p + 1); pz[i] = __ldg(p + 2); }
            }
            urow[i] = a.uf ? a.uf + ((size_t)bi * a.n + jn[i]) * C1 : nullptr;
            if constexpr (kHoldU) {
                if (a.uf != nullptr) {
#pragma unroll
                    for (int q = 0; q < kUH; ++q) uh[i][q] = __ldg(reinterpret_cast<const float2*>(urow[i] + 8 * q + 2 * t));
                }
            }
        }
    };

    // The chunk after the current one is claimed at the top of the current one's first pass into the other table, read after
    // the first barrier of the current one's end and its slot counts filled before the second; the barriers order the read
    // before the next claim and the table before the gather that reads it.  The current chunk is read from its table where
    // it is needed rather than held in a register through the pass (a spilled word in SA1 and SA2).
    if (ut == 0) s_chunk[unit][0] = atomicAdd(a.tile_counter, 1u);
    unit_bar_sync(ubar, uthreads);
    if (s_chunk[unit][0] < nchunks) fill_table(s_chunk[unit][0], 0);
    unit_bar_sync(ubar, uthreads);
    int buf = 0, p = 0;                                       // table and pass index of the current chunk
    if (kAhead && s_chunk[unit][0] < nchunks) { gather_a(s_chunk[unit][0], 0, 0); gather_b(); }
    uint32_t it = 0;                                          // passes of this unit
    for (; s_chunk[unit][buf] < nchunks; ++it) {
        if (p == 0 && ut == 0) s_chunk[unit][buf ^ 1] = atomicAdd(a.tile_counter, 1u);
        SA_STAMP(it, kSaTop);
        if (!kAhead) { gather_a(s_chunk[unit][buf], buf, p); gather_b(); }
        SA_STAMP_AFTER(it, kSaInputs, kHoldU ? uh[0][0].x : a.uf == nullptr ? px[0] : __ldg(urow[0] + 2 * t));

        // ---- layer 1 on the FMA pipe, straight into the A fragments (K = C1) ----
        uint32_t A[NP][8][4];
        if (a.uf != nullptr) {
            // V[j] + c . w1c: the centre term of a column is shared by this thread's two rows (one neighbourhood per warp)
#pragma unroll
            for (int s = 0; s < C1 / 16; ++s) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int k = 16 * s + 8 * h + 2 * t;
                    const float2 cwx = *reinterpret_cast<const float2*>(w1c + k), cwy = *reinterpret_cast<const float2*>(w1c + C1 + k),
                                 cwz = *reinterpret_cast<const float2*>(w1c + 2 * C1 + k);
                    const float2 ct = ffma2_rn(make_float2(cz, cz), cwz, ffma2_rn(make_float2(cy, cy), cwy, fmul2_rn(make_float2(cx, cx), cwx)));
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        float2 v;
                        if constexpr (kHoldU) v = uh[i][2 * s + h];
                        else v = __ldg(reinterpret_cast<const float2*>(urow[i] + k));
                        v = fadd2_rn(v, ct);
                        if (a.relu1) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
                        put_a<NP, 8>(A, s, i + 2 * h, v.x, v.y, ovf);
                    }
                }
            }
        } else {
            // t + (x_j - c) . w1x (+ c . w1c)
            float dx[2], dy[2], dz[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                if constexpr (kHoldU) { dx[i] = uh[i][0].x - cx; dy[i] = uh[i][0].y - cy; dz[i] = uh[i][1].x - cz; }
                else { dx[i] = px[i] - cx; dy[i] = py[i] - cy; dz[i] = pz[i] - cz; }
            }
#pragma unroll
            for (int s = 0; s < C1 / 16; ++s) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int k = 16 * s + 8 * h + 2 * t;
                    const float2 sh = *reinterpret_cast<const float2*>(t1 + k);
                    const float2 wx = *reinterpret_cast<const float2*>(w1x + k), wy = *reinterpret_cast<const float2*>(w1x + C1 + k),
                                 wz = *reinterpret_cast<const float2*>(w1x + 2 * C1 + k);
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        float2 v = sh;
                        if (a.w1c != nullptr) {            // EdgeConv: the part of the first layer that acts on the centre x_i
                            const float2 cwx = *reinterpret_cast<const float2*>(w1c + k), cwy = *reinterpret_cast<const float2*>(w1c + C1 + k),
                                         cwz = *reinterpret_cast<const float2*>(w1c + 2 * C1 + k);
                            v = ffma2_rn(make_float2(cz, cz), cwz, ffma2_rn(make_float2(cy, cy), cwy, ffma2_rn(make_float2(cx, cx), cwx, v)));
                        }
                        v = ffma2_rn(make_float2(dz[i], dz[i]), wz, ffma2_rn(make_float2(dy[i], dy[i]), wy, ffma2_rn(make_float2(dx[i], dx[i]), wx, v)));
                        if (a.relu1) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
                        put_a<NP, 8>(A, s, i + 2 * h, v.x, v.y, ovf);
                    }
                }
            }
        }
        SA_STAMP(it, kSaLayer1);

        if constexpr (NL == 2) {
            // ---- inner layer (N0 wide): D fragments -> affine + ReLU -> A fragments of the last layer ----
            constexpr int NCH = N0 / 64;
            float d[NCH][32];
            sa_mma_issue<NP, C1 / 16, NCH>(d, A, smem_u32(base + L.w[0]), (uint32_t)(C1 / 64) * bb);
            SA_STAMP(it, kSaL2Issued);
            wg_wait_all();
#pragma unroll
            for (int c = 0; c < NCH; ++c) wg_fence_acc(d[c]);
            SA_STAMP(it, kSaL2Retired);
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int j = 2 * jj + h, col = c * 64 + 8 * j + 2 * t;
                        const float sc0 = sl0[col], sc1 = sl0[col + 1], sh0 = tl0[col], sh1 = tl0[col + 1];
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            float v0 = fmaf(d[c][4 * j + 2 * i], sc0, sh0), v1 = fmaf(d[c][4 * j + 2 * i + 1], sc1, sh1);
                            if (a.relu[0]) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                            put_a<NP, 8>(A, c * 4 + jj, i + 2 * h, v0, v1, ovf);
                        }
                    }
                }
            }
            SA_STAMP(it, kSaL2Epi);
        }
        if constexpr (NP == 2) {                              // every leading piece is stored; the flag is raised at once, so
            if (f16x2_overflowed(ovf)) atomicOr(a.ovf, 1u);   // that no predicate is held through the rest of the pass
            ovf = 0u;
        }
        {
            // ---- last layer, 64 output channels at a time, max-pooled over each neighbourhood in the unit's pooling buffer ----
            // kDouble: chunk nc + 1's group is issued before chunk nc's epilogue and runs during it (wait_group 1)
            const int N = a.Ntot[last];
            const int NG = a.stream_last ? 1 : NCL;           // 64-channel chunks per store: a streamed layer's ring slot holds one
            // the next pass continues this chunk, or opens the one in the other table (a joint chunk is one pass: never `same`)
            const bool same = (p + 1) * W < slot_total();
            // gather the next pass of this chunk in the shadow of this one's last layer; the first pass of a chunk gathers after
            // the store that ends the chunk before, which fills its slot table
            const bool ahead = kAhead && same;
            auto issue = [&](float (&acc)[1][32], int nc) {
                uint32_t wb;
                if (a.stream_last) {                              // ring use q = chunk nc of pass it (every pass runs all NCL)
                    const uint32_t q = it * (uint32_t)NCL + (uint32_t)nc;
                    mbar_wait(&s_wbar[q & 1], (q >> 1) & 1u);
                    wb = smem_u32(base + L.ring[q & 1]);
                } else {
                    wb = smem_u32(base + L.w[last]) + (uint32_t)(nc * (KSL / 4)) * bb;
                }
                sa_mma_issue<NP, KSL, 1>(acc, A, wb, 0u);
                SA_STAMP(it, kSaChunk0 + 3 * nc);
            };
            // affine + ReLU of chunk nc, this warp's 16-row column maxima folded into its neighbourhood's row.  Every warp folds,
            // those past the chunk's last slot included (they repeat that slot), so that no branch sits inside the wgmma group
            // in flight
            auto epilogue = [&](float (&acc)[1][32], int nc) {
                wg_fence_acc(acc[0]);
                SA_STAMP(it, kSaChunk0 + 3 * nc + 1);
                auto rowmax = [&](int j) {                        // columns 8j + 2t, + 1: max over rows g, g + 8
                    const int col = nc * 64 + 8 * j + 2 * t;
                    const float2 sc = *reinterpret_cast<const float2*>(slL + col), sh = *reinterpret_cast<const float2*>(tlL + col);
                    float lo0 = fmaf(acc[0][4 * j], sc.x, sh.x), hi0 = fmaf(acc[0][4 * j + 2], sc.x, sh.x);
                    float lo1 = fmaf(acc[0][4 * j + 1], sc.y, sh.y), hi1 = fmaf(acc[0][4 * j + 3], sc.y, sh.y);
                    if (a.relu[last]) { lo0 = fmaxf(lo0, 0.f); hi0 = fmaxf(hi0, 0.f); lo1 = fmaxf(lo1, 0.f); hi1 = fmaxf(hi1, 0.f); }
                    return make_float2(fmaxf(lo0, hi0), fmaxf(lo1, hi1));
                };
                float v[8];
                const bool up = (g >> 2) & 1;
#pragma unroll
                for (int j = 0; j < 4; ++j) {                     // first step of the butterfly: column blocks j and j + 4
                    const float2 lo = rowmax(j), hi = rowmax(j + 4);
                    v[2 * j] = fmaxf(up ? hi.x : lo.x, __shfl_xor_sync(0xffffffffu, up ? lo.x : hi.x, 16));
                    v[2 * j + 1] = fmaxf(up ? hi.y : lo.y, __shfl_xor_sync(0xffffffffu, up ? lo.y : hi.y, 16));
                }
                colmax_halve<4>(v, (g >> 1) & 1);
                colmax_halve<2>(v, g & 1);
                // this warp's columns 8g + 2t, + 1 of its neighbourhood's row (found again here rather than held through the pass)
                const uint32_t dst = smem_u32(base + pool) + 4u * (uint32_t)(slot_nb(p) * PC + (a.stream_last ? 0 : nc * 64) + 8 * g + 2 * t);
                red_smem_max(dst, sa_pool_code(v[0]));
                red_smem_max(dst + 4u, sa_pool_code(v[1]));
                SA_STAMP(it, kSaChunk0 + 3 * nc + 2);
            };
            // the end of a chunk of neighbourhoods (streamed: of its 64 channels from c0 on): the buffer's rows are stored for the
            // neighbourhoods before a.groups (each of them has a slot, so its row holds a value) and reset, two columns per thread.
            // The last store of the pass fills the next chunk's table and gathers its first pass; not an earlier one, whose
            // gather would move the prefix that the pass's later epilogues find their rows with
            auto store = [&](int c0) {
                unit_bar_sync(ubar, uthreads);                    // every warp's atomics have landed; ring slot consumed
                SA_STAMP(it, kSaEnd1);
                const unsigned next = s_chunk[unit][buf ^ 1];     // claimed at the top of this chunk's first pass
                const bool last_store = c0 + NG == NCL;
                if (last_store && next < nchunks) fill_table(next, buf ^ 1);
                if (a.stream_last && tid == 0)                    // ring use c0 of this pass is consumed
                    sa_fill_ring(it * (uint32_t)NCL + (uint32_t)c0 + 2u, a.image[last], NCL, L, base, s_wbar);
                const long long g0 = (long long)s_chunk[unit][buf] * C;
                const int rows = (int)min((long long)C, a.groups - g0), half = PC / 2;
                for (int e = ut; e < C * half; e += uthreads) {
                    int2* const q = reinterpret_cast<int2*>(base + pool) + e;
                    const int r = e / half, col = c0 * 64 + 2 * (e - r * half);
                    if (r < rows) {
                        const int2 c = *q;
                        *reinterpret_cast<float2*>(a.out + (size_t)(g0 + r) * N + col) = make_float2(sa_pool_value(c.x), sa_pool_value(c.y));
                    }
                    *q = make_int2(kSaPoolEmpty, kSaPoolEmpty);
                }
                unit_bar_sync(ubar, uthreads);                    // the rows are reset; the next chunk's slot table is filled
                SA_STAMP(it, kSaEnd2);
                if (kAhead && last_store && next < nchunks) {
                    gather_a(next, buf ^ 1, 0);
                    SA_STAMP(it, kSaNextA);
                    gather_b();
                    SA_STAMP(it, kSaNextB);
                }
            };
            // Every path below issues and waits in straight lines, and every group ends in wait_group 0 before the store: ptxas
            // keeps the wgmma asynchronous only when it can see which group a wait retires on every path.  Stage B of the
            // gather is issued on every path that waits for the last chunk (NCL - 1), before that wait and after the epilogue
            // of the chunk before it, so it follows stage A in every pass that gathers ahead.
            float d0[1][32];
            for (int c0 = 0; c0 < NCL; c0 += NG) {
                const int end = c0 + NG;
                issue(d0, c0);
                if (ahead && c0 == 0) {
                    gather_a(s_chunk[unit][buf], buf, p + 1);
                    SA_STAMP(it, kSaNextA);
                }
                if constexpr (kDouble) {
                    float d1[1][32];
                    int nc = c0;
                    for (; nc + 2 < end; nc += 2) {
                        issue(d1, nc + 1); wg_wait<1>(); epilogue(d0, nc);
                        issue(d0, nc + 2); wg_wait<1>(); epilogue(d1, nc + 1);
                    }
                    if (nc + 1 < end) {
                        issue(d1, nc + 1); wg_wait<1>(); epilogue(d0, nc);
                        if (ahead && nc + 2 == NCL) { gather_b(); SA_STAMP(it, kSaNextB); }
                        wg_wait<0>(); epilogue(d1, nc + 1);
                    } else {
                        if (ahead && nc + 1 == NCL) { gather_b(); SA_STAMP(it, kSaNextB); }
                        wg_wait<0>(); epilogue(d0, nc);
                    }
                } else {
                    for (int nc = c0;;) {
                        if (ahead && nc + 1 == NCL) { gather_b(); SA_STAMP(it, kSaNextB); }
                        wg_wait<0>(); epilogue(d0, nc);
                        if (++nc == end) break;
                        issue(d0, nc);
                    }
                }
                if (!same) store(c0);
            }
            if (!same) { buf ^= 1; p = 0; }
            else ++p;
        }
    }
    if constexpr (NP == 2) {
        if (tid == 0)
            for (int l = 0; l < NL; ++l)
                if (a.wflag[l] != nullptr && *a.wflag[l] != 0u) atomicOr(a.ovf, 1u);
    }
    if (tid == 0 && a.stream_last)                                    // the two fills issued ahead must land before the CTA exits
        for (uint32_t q = it * (uint32_t)NCL; q < it * (uint32_t)NCL + 2u; ++q) mbar_wait(&s_wbar[q & 1], (q >> 1) & 1u);
}

// ------------------------------------------------------------------------------------------------------------------
// Dense layer on the tensor cores: out = relu?((x . W [+ xyz3 . w3]) * scale + shift), optional max over runs of pool_k rows.
// ------------------------------------------------------------------------------------------------------------------
struct TcDenseArgs {
    long long rows;
    int K, Kp, N;          // Kp = K rounded up to 64
    int pool_k;            // 1, 32, 64 or a multiple of 128
    int relu;
    const float* x;        // (rows, K)
    const float* scale;    // (N) or null
    const float* shift;    // (N) or null
    const float* xyz3;     // optional side input (rows, 3): out += xyz3 . w3 before scale/shift (the xyz rows of a
    const float* w3;       // (3, N)                          [xyz, features] . W product, kept off the K loop)
    float* out;
    // training-mode forward: the input is relu(x * in_scale + in_shift) per INPUT channel (the previous layer's
    // batch norm, applied while the operand is staged) and per-tile column statistics of the stored values are written
    const float* in_scale = nullptr;   // (K) or null
    const float* in_shift = nullptr;
    int in_relu = 0;
    float* stat_partial = nullptr;     // (row tiles, 2, N) or null
    // optional per-row-group input (pool_k == 1): row r adds group_add[r / group_rows] (N) before scale/shift, e.g. the
    // per-cloud product of a global feature tiled over the cloud's points
    const float* group_add = nullptr;
    long long group_rows = 0;
    RingArgs ring;                     // W (Kp, N) in the format of NP, tile width 64 NC
};

// The dense layer on the ring (ring_gemm.cuh), unit = 128-row tile x Nt = 64 NC-column tile, all Kp / 64 K blocks, claimed from
// the launch's counter.  The producers stage x rows, 16 bytes per copy, or 4 for K % 4 != 0 / unaligned x; the consumers read rows
// past `rows` and columns past K as zero.  Each unit's affine goes through shared memory, loaded once per column under the K loop:
// fp16x2 folds the column factor 2^-e_n into the scale, and its inverse brings what the epilogue adds to the accumulators into their
// units.  Epilogue in the fragment layout: xyz side input, per-group input, affine, ReLU, then either float2 stores (+ per-tile
// column statistics) or the max over pool_k rows; the cross-warp part synchronises the consumers on named barrier 1.
template <int NP, int NC>
struct DenseOp {
    static constexpr int Nt = 64 * NC;
    const TcDenseArgs& a;
    static constexpr bool kClaim = true;
    static constexpr uint32_t kBudget = 210u * 1024u;         // four stages at NP = 2, NC = 1, next to Smem
    struct Smem {
        float red[2][8][Nt];                                  // per warp: column sums and sums of squares, or column maxima
        __align__(16) float aff[2][3][Nt];                    // [unit parity]: scale x column factor, shift, 1 / column factor
    };
    struct Unit {
        int nb, col0, par;
        long long tile;                                       // row tile
        long long r[2];
        bool v[2];
    };

    __device__ int units(int) const { return (int)((a.rows + 127) / 128 * (a.N / Nt)); }

    template <class Put>
    __device__ void produce(int unit, int, int pw, int lane, Smem&, Put&& put) const {
        const int NTC = a.N / Nt, KC = a.Kp / 64;
        const long long row0 = (long long)(unit / NTC) * 128;
        const int nt = unit % NTC, r0 = 32 * pw, nr = (int)max(0LL, min(32LL, a.rows - row0 - r0));
        if ((a.K & 3) == 0 && (reinterpret_cast<uintptr_t>(a.x) & 15) == 0) {     // rows of x are 16-byte aligned
            for (int kb = 0; kb < KC; ++kb) put((size_t)nt * KC + kb, [&](uint32_t xs) { stage_rows16(xs, a.x, a.K, row0, r0, nr, kb, a.K, lane); });
            return;
        }
        for (int kb = 0; kb < KC; ++kb)
            put((size_t)nt * KC + kb, [&](uint32_t xs) {
#pragma unroll 1
                for (int e = lane; e < nr * 64; e += 32) {
                    const int row = r0 + (e >> 6), c = e & 63;
                    if (kb * 64 + c < a.K) cp_async4(xs + (uint32_t)row * kRingXRow + (uint32_t)c * 4u, a.x + (size_t)(row0 + row) * a.K + kb * 64 + c);
                }
            });
    }

    // the unit's affine into aff[n & 1]: the write for this unit follows the barrier of the last one, so it cannot overtake the
    // epilogue of the unit before
    __device__ Unit unit(int unit, int, int row, Smem& sm, int n) const {
        const int NTC = a.N / Nt, tid = threadIdx.x;
        Unit u;
        u.nb = a.Kp / 64;
        u.tile = unit / NTC;
        u.col0 = unit % NTC * Nt;
        u.par = n & 1;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            u.r[i] = u.tile * 128 + row + 8 * i;
            u.v[i] = u.r[i] < a.rows;
        }
        if (tid < Nt) {
            const int col = u.col0 + tid;
            const float cs = NP == 2 ? __ldg(a.ring.colscale + col) : 1.f;
            sm.aff[u.par][0][tid] = (a.scale ? __ldg(a.scale + col) : 1.f) * cs;
            sm.aff[u.par][1][tid] = a.shift ? __ldg(a.shift + col) : 0.f;
            sm.aff[u.par][2][tid] = NP == 2 ? pow2_rcp(cs) : 1.f;
        }
        return u;
    }

    // the row and K masks, then the previous layer's batch norm + ReLU of training mode
    __device__ void load(const Unit& u, const float* xs, int kb, int t, float2 (&x)[4][2][2]) const {
#pragma unroll
        for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int k = kb * 64 + 16 * s + 8 * h + 2 * t;
                    float2 v = make_float2(0.f, 0.f);
                    if (u.v[i]) {
                        const float2 y = staged_pair(xs, s, h, i, t);
                        if (k < a.K) v.x = y.x;
                        if (k + 1 < a.K) v.y = y.y;
                        if (a.in_scale != nullptr) {
                            if (k < a.K) { v.x = fmaf(v.x, __ldg(a.in_scale + k), __ldg(a.in_shift + k)); if (a.in_relu) v.x = fmaxf(v.x, 0.f); }
                            if (k + 1 < a.K) { v.y = fmaf(v.y, __ldg(a.in_scale + k + 1), __ldg(a.in_shift + k + 1)); if (a.in_relu) v.y = fmaxf(v.y, 0.f); }
                        }
                    }
                    x[s][h][i] = v;
                }
    }

    // One 64-column chunk.  Its cross-warp fold reads the chunk's own columns of `red`, so the next chunk's writes need no barrier;
    // the next unit's writes follow the barrier in front of its first chunk.
    __device__ void epilogue(const Unit& u, float (&acc)[32], int col0, int t, const float*, Smem& sm) const {
        const int tid = threadIdx.x, warp = tid >> 5, g = (tid & 31) >> 2, cl0 = col0 - u.col0;
        const float (&aff)[3][Nt] = sm.aff[u.par];
        if (cl0 == 0) unit_bar_sync(1, kRingConsumers);        // the unit's affine is in `aff`
        float xs[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
        if (a.xyz3 != nullptr)
#pragma unroll
            for (int i = 0; i < 2; ++i)
                if (u.v[i])
#pragma unroll
                    for (int k = 0; k < 3; ++k) xs[i][k] = __ldg(a.xyz3 + (size_t)u.r[i] * 3 + k);
        // the per-group input, added to the accumulators in a pass of its own so that the loop below is the same code with or
        // without it.  Rows g and g + 8 may lie in different groups, and groups need not align with the 128-row tiles.  fp16x2:
        // the accumulators hold the product times 2^e_n, and so must what is added to them (exact, the rounding of the sum is
        // that of the unscaled one)
        if (a.group_add != nullptr)
#pragma unroll
            for (int i = 0; i < 2; ++i)
                if (u.v[i]) {
                    const float* ga = a.group_add + (size_t)(u.r[i] / a.group_rows) * a.N + col0 + 2 * t;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float2 gv = __ldg(reinterpret_cast<const float2*>(ga + 8 * j));
                        const float2 f = *reinterpret_cast<const float2*>(&aff[2][cl0 + 8 * j + 2 * t]);
                        acc[4 * j + 2 * i] = fmaf(gv.x, f.x, acc[4 * j + 2 * i]);
                        acc[4 * j + 2 * i + 1] = fmaf(gv.y, f.y, acc[4 * j + 2 * i + 1]);
                    }
                }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int cl = cl0 + 8 * j + 2 * t;
            float y[2][2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = u.col0 + cl + e;
                const float sc = aff[0][cl + e], sh = aff[1][cl + e];
                float w0 = 0.f, w1 = 0.f, w2 = 0.f;
                if (a.xyz3 != nullptr) {
                    const float f = aff[2][cl + e];
                    w0 = __ldg(a.w3 + col) * f; w1 = __ldg(a.w3 + a.N + col) * f; w2 = __ldg(a.w3 + 2 * a.N + col) * f;
                }
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    float x = acc[4 * j + 2 * i + e];
                    if (a.xyz3 != nullptr) x = fmaf(xs[i][2], w2, fmaf(xs[i][1], w1, fmaf(xs[i][0], w0, x)));
                    x = fmaf(x, sc, sh);
                    if (a.relu) x = fmaxf(x, 0.f);
                    y[i][e] = x;
                }
            }
            if (a.pool_k == 1) {
#pragma unroll
                for (int i = 0; i < 2; ++i)
                    if (u.v[i]) *reinterpret_cast<float2*>(a.out + (size_t)u.r[i] * a.N + u.col0 + cl) = make_float2(y[i][0], y[i][1]);
                if (a.stat_partial != nullptr) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float ssum = 0.f, ssq = 0.f;
#pragma unroll
                        for (int i = 0; i < 2; ++i)
                            if (u.v[i]) { ssum += y[i][e]; ssq = fmaf(y[i][e], y[i][e], ssq); }
                        ssum = warp_rowsum16(ssum);
                        ssq = warp_rowsum16(ssq);
                        if (g == 0) { sm.red[0][warp][cl + e] = ssum; sm.red[1][warp][cl + e] = ssq; }
                    }
                }
            } else {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float m = warp_rowmax16(u.v[0] ? y[0][e] : -FLT_MAX, u.v[1] ? y[1][e] : -FLT_MAX);
                    if (g == 0) sm.red[0][warp][cl + e] = m;
                }
            }
        }
        if (a.pool_k == 1) {
            if (a.stat_partial != nullptr) {
                // per-tile column statistics, the eight warps' 16-row partials folded in warp order (deterministic)
                unit_bar_sync(1, kRingConsumers);
                if (tid < 64) {
                    const int cl = cl0 + tid;
                    float t0 = 0.f, t1 = 0.f;
                    for (int w = 0; w < 8; ++w) { t0 += sm.red[0][w][cl]; t1 += sm.red[1][w][cl]; }
                    float* dst = a.stat_partial + (size_t)u.tile * 2 * a.N;
                    dst[u.col0 + cl] = t0;
                    dst[a.N + u.col0 + cl] = t1;
                }
            }
        } else {
            unit_bar_sync(1, kRingConsumers);
            const bool big = a.pool_k > 128;                             // the whole 128-row tile lies inside one group
            const int wpg = big ? 8 : a.pool_k / 16;                     // warps per pooling group
            for (int e = tid; e < (8 / wpg) * 64; e += kRingConsumers) {
                const int grp = e / 64, cl = cl0 + e % 64;
                const long long rs = u.tile * 128 + grp * wpg * 16;
                if (rs >= a.rows) continue;
                float mx = sm.red[0][grp * wpg][cl];
                for (int w = 1; w < wpg; ++w) mx = fmaxf(mx, sm.red[0][grp * wpg + w][cl]);
                const long long wg = rs / a.pool_k;
                if (!big) {
                    a.out[(size_t)wg * a.N + u.col0 + cl] = mx;
                } else {
                    int code = __float_as_int(mx);
                    code = code >= 0 ? code : code ^ 0x7fffffff;
                    atomicMax(reinterpret_cast<int*>(a.out) + (size_t)wg * a.N + u.col0 + cl, code);
                }
            }
        }
    }
};

template <int NP, int NC>
__global__ void __launch_bounds__(kRingThreads, 1) tc_dense_kernel(const __grid_constant__ TcDenseArgs a) {
    ring_gemm<NP, NC>(DenseOp<NP, NC>{a}, a.ring);
}

static_assert(ring_stages(2, 1, DenseOp<2, 1>::kBudget) == 4 && ring_stages(3, 1, DenseOp<3, 1>::kBudget) == 3 &&
              ring_stages(2, 2, DenseOp<2, 2>::kBudget) == 3 && ring_stages(3, 2, DenseOp<3, 2>::kBudget) == 2, "stages of the dense ring");
static const RingKernels kDenseRing = {{{(const void*)tc_dense_kernel<2, 1>, (const void*)tc_dense_kernel<2, 2>},
                                        {(const void*)tc_dense_kernel<3, 1>, (const void*)tc_dense_kernel<3, 2>}},
                                       "tc_dense_kernel", DenseOp<2, 1>::kBudget};

static bool tc_dense_eligible(long long rows, int K, int N, int pool_k) {
    if (rows < 128 || K < 32 || N < 64 || (N % 64) != 0) return false;
    if (N > 64 && (N % 128) != 0) return false;
    if (!(pool_k == 1 || pool_k == 32 || pool_k == 64 || (pool_k >= 128 && pool_k % 128 == 0))) return false;
    if (pool_k > 1 && rows % pool_k != 0) return false;
    return true;
}

// Operand split of the inference launches: 2 = fp16x2 with the np = 3 rerun guard (default), 3 = bf16x3 only (psa_set_mlp_mode(2)).
static std::atomic<int> g_tc_np{2};        // process-wide settings: atomics, so that a concurrent psa_set_mlp_mode is a race-free (if unordered) switch
static std::atomic<int> g_mlp_mode{0};
int tc_np() { return g_tc_np; }
int mlp_mode() { return g_mlp_mode; }

// Workspace reservation for one dense layer's images: an fp16x2 image (used when the caller brought no prebuilt one) followed by
// the bf16x3 image of the guarded rerun / of mode 2 / of the training forward.
static size_t tc_dense_image_off3(int K, int N) { return tc_image_alloc_bytes((K + 63) & ~63, N, 2); }
size_t tc_dense_image_bytes(int K, int N) { return tc_dense_image_off3(K, N) + tc_image_alloc_bytes((K + 63) & ~63, N, 3); }

// bytes of a prebuilt image of the current split: mode 0 = fp16x2 blocks + their bf16x3 twin, mode 2 = bf16x3 blocks
static size_t tc_plan_image_bytes(int Kp, int N) { return g_tc_np == 2 ? tc_image_alloc_bytes(Kp, N, 2) + tc_image_alloc_bytes(Kp, N, 3) : tc_image_alloc_bytes(Kp, N, 3); }

// tile width of a dense layer (and of its weight image), with the format flag of the current split: 128 when N allows it and
// 128-wide tiles keep more than half of the SMs busy (one persistent CTA per SM), else 64.  Narrow tiles read x once per 64
// channels instead of once per 128: measured on SA3 (H100), 64-wide won for 64 tiles of 128 (layer 0) and lost for 128 (layer 1).
int tc_dense_nt(long long rows, int N) {
    const bool wide = (N % 128) == 0 && 2 * ((rows + 127) / 128 * (N / 128)) > kNumSMs;
    return (wide ? 128 : 64) | image_flag(g_tc_np);
}

// builds the image of W (K x N, rows K..Kp zero) in the format `Nt` carries (width | format flag); fp16x2: zeroes the trailer and
// computes the column factors first
int build_image(int K, int Kp, int N, int Nt, const float* W, uint8_t* image, cudaStream_t st, const unsigned int* run_if) {
    if (Nt & kImageF16x2) {
        unsigned int* trailer = reinterpret_cast<unsigned int*>(image + tc_image_trailer_off(Kp, N, 2));
        float* colscale = reinterpret_cast<float*>(image + tc_image_colscale_off(Kp, N, 2));
        PSA_CUDA(cudaMemsetAsync(trailer, 0, 256, st));
        tc_col_scale_kernel<<<(N + 31) / 32, dim3(32, 8), 0, st>>>(K, N, W, colscale, trailer);
        int rc = check_launch("tc_col_scale_kernel");
        if (rc != PSA_OK) return rc;
        tc_prep_weights_kernel<2><<<(Kp * N + 255) / 256, 256, 0, st>>>(K, Kp, N, Nt & ~kImageFlags, W, colscale, image, run_if);
    } else {
        tc_prep_weights_kernel<3><<<(Kp * N + 255) / 256, 256, 0, st>>>(K, Kp, N, Nt & ~kImageFlags, W, nullptr, image, run_if);
    }
    return check_launch("tc_prep_weights_kernel");
}
const unsigned int* image_trailer(const uint8_t* image, int Kp, int N) {
    return reinterpret_cast<const unsigned int*>(image + tc_image_trailer_off(Kp, N, 2));
}
const float* image_colscale(const uint8_t* image, int Kp, int N) {
    return reinterpret_cast<const float*>(image + tc_image_colscale_off(Kp, N, 2));
}

static long long tc_dense_units(long long rows, int N, int Nt) { return (rows + 127) / 128 * (N / Nt); }

// The zeroed 256-byte word region of an inference entry point.  Its dense step l -- layer l of a chain, the U GEMM (0) and the
// level (1) of tc_sa_run, EdgeConv's GEMM (0) -- has its range flag at [l] (np = 2: raised when a value left the fp16 range; the
// bf16x3 rerun is conditional on it) and the tile counters of its launch and of its rerun at [PSA_MAX_MLP_LAYERS + 2 l, + 1].
struct StepWords {
    unsigned int* flag;
    unsigned int* counters;
};
static StepWords step_words(unsigned int* region, int l) { return {region + l, region + PSA_MAX_MLP_LAYERS + 2 * l}; }
constexpr int kClusterFlagStep = 3;        // the group-all cluster kernel's flag: a step its three-layer chain leaves free

// One inference dense layer: out = relu?((x . W [+ xyz3 . w3] [+ group_add[r / group_rows]]) * scale + shift), optional max over
// runs of pool_k rows (not with group_add).
struct DenseStep {
    long long rows;
    int K, N, pool_k, relu;
    const float* x;
    const float* W;
    const float* scale;                  // or null
    const float* shift;                  // or null
    float* out;
    const float* xyz3 = nullptr;         // (rows, 3) side input with w3 (3, N)
    const float* w3 = nullptr;
    const float* group_add = nullptr;
    long long group_rows = 0;
    const uint8_t* prebuilt = nullptr;   // image of W in the current split's format (psa_prepare_weight_image), or null
    uint8_t* img = nullptr;              // tc_dense_image_bytes(K, N) of scratch: the images not prebuilt are built here
    StepWords words{};                   // in a zeroed word region
    float* fc_partial = nullptr;         // non-null: fc_small's partial sums, for an FMA layer of rows <= 32
};

// The one choice between the tensor cores and the FMA kernels of an inference dense layer: mode 1 never takes the tensor cores.
static bool dense_on_tc(long long rows, int K, int N, int pool_k) { return g_mlp_mode != 1 && tc_dense_eligible(rows, K, N, pool_k); }

// a tensor-core step's kernel arguments (`ring` is filled by ring_run / ring_rerun) and weights
static TcDenseArgs tc_dense_args(const DenseStep& s) {
    TcDenseArgs a;
    a.rows = s.rows; a.K = s.K; a.Kp = (s.K + 63) & ~63; a.N = s.N; a.pool_k = s.pool_k; a.relu = s.relu;
    a.x = s.x; a.scale = s.scale; a.shift = s.shift; a.out = s.out; a.xyz3 = s.xyz3; a.w3 = s.w3;
    a.group_add = s.group_add; a.group_rows = s.group_rows;
    return a;
}
static RingWeights tc_dense_weights(const DenseStep& s) {
    return RingWeights{s.K, (s.K + 63) & ~63, s.N, tc_dense_nt(s.rows, s.N) & ~kImageFlags, s.W, s.img, s.img + tc_dense_image_off3(s.K, s.N), s.prebuilt};
}

static int run_dense(const DenseStep& s, cudaStream_t st) {
    if (dense_on_tc(s.rows, s.K, s.N, s.pool_k)) {
        RingPool pool;
        if (s.pool_k > 128) { pool.out = s.out; pool.count = s.rows / s.pool_k * s.N; }
        const RingWeights w = tc_dense_weights(s);
        return ring_run(kDenseRing, tc_dense_args(s), tc_dense_units(s.rows, s.N, w.Nt), w, s.words.flag, s.words.counters, st, pool);
    }
    DenseArgs d;
    d.rows = s.rows; d.K = s.K; d.N = s.N; d.pool_k = s.pool_k; d.relu = s.relu;
    d.x = s.x; d.W = s.W; d.scale = s.scale; d.shift = s.shift; d.out = s.out;
    d.group_add = s.group_add; d.group_rows = s.group_rows; d.xyz3 = s.xyz3; d.w3 = s.w3;
    if (s.fc_partial != nullptr && s.rows <= 32 && s.pool_k == 1 && s.group_add == nullptr && s.xyz3 == nullptr) return launch_fc_small(d, s.fc_partial, st);
    return launch_dense(d, st);
}

// Training-mode forward of one layer on tc_dense_kernel: y = relu(bn_prev(x)) . W + bias (pre-BN output), per-row-tile column
// statistics.  The weights change every step, so the image is rebuilt into `image_ws` (tc_dense_image_bytes(K, N)) per call.
// bf16x3 only: batch-statistics activations are not range-checked.  No zeroed word comes with the call: the tiles are taken in
// a static order.
bool tc_train_fwd_eligible(long long rows, int K, int N) {
    // pays off from two K blocks up (K = 64 layers stay on the fp32 FMA kernel)
    return rows >= 128 && K >= 128 && K <= 512 && N >= 128 && (N % 128) == 0;
}
int launch_tc_dense_train(long long rows, int K, int N, const float* x, const float* in_scale, const float* in_shift, int in_relu,
                          const float* W, const float* bias, float* y, float* stat_partial, uint8_t* image_ws, cudaStream_t st) {
    const int Kp = (K + 63) & ~63;
    int rc = build_image(K, Kp, N, 128 | kImageBf16x3, W, image_ws, st);
    if (rc != PSA_OK) return rc;
    TcDenseArgs a;
    a.rows = rows; a.K = K; a.Kp = Kp; a.N = N; a.pool_k = 1; a.relu = 0;
    a.x = x; a.scale = nullptr; a.shift = bias; a.out = y; a.xyz3 = nullptr; a.w3 = nullptr;
    a.in_scale = in_scale; a.in_shift = in_shift; a.in_relu = in_relu; a.stat_partial = stat_partial;
    a.ring.image = image_ws;
    return ring_launch(kDenseRing, 3, 128, &a, tc_dense_units(rows, N, 128), st);
}

// A prebuilt image (psa_prepare_weight_image) is used when its format, tile width and first row match; otherwise null (the
// launchers then build what they need in their workspace).  `Nt` carries the format flag.
static const uint8_t* prebuilt_image(const psa_mlp* mlp, int l, int row0, int Nt) {
    if (mlp->image[l] != nullptr && mlp->image_nt[l] == Nt && mlp->image_row0[l] == row0) return reinterpret_cast<const uint8_t*>(mlp->image[l]);
    return nullptr;
}

// Can this MLP / geometry run on the tensor-core kernel with `np` pieces per operand?  (otherwise the fp32-FMA fused kernel
// in mlp.cu is used).  Whatever fits with three pieces fits with two; the guarded default needs both.
bool tc_sa_eligible(const psa_mlp* mlp, int c, int nsample, TcArgs* out, int np) {
    if (mlp->n_layers < 2 || mlp->n_layers > 1 + kMaxTcLayers) return false;
    if (!(nsample == 32 || nsample == 64 || nsample == 128)) return false;
    if (mlp->channels[0] != 3 + c) return false;
    const int C1 = mlp->channels[1];
    if (!(C1 == 64 || C1 == 128)) return false;
    TcArgs a{};
    a.C1 = C1;
    a.nl = mlp->n_layers - 1;
    a.np = np;
    for (int l = 0; l < a.nl; ++l) {
        a.Kd[l] = mlp->channels[1 + l];
        a.Ntot[l] = mlp->channels[2 + l];
        if (!(a.Kd[l] == 64 || a.Kd[l] == 128)) return false;
        const bool is_last = (l == a.nl - 1);
        if (!is_last && !(a.Ntot[l] == 64 || a.Ntot[l] == 128)) return false;       // D and the next A operand are one tile wide
        if (is_last && !(a.Ntot[l] == 64 || a.Ntot[l] % 128 == 0)) return false;
    }
    // the last layer is streamed in 64-channel chunks if it does not fit next to the others; a level that does not fit even then
    // runs on the fp32-FMA fused kernel
    a.stream_last = 0;
    if (tc_sa_layout(a).total + 1024 > kSmemBudget) a.stream_last = 1;
    if (tc_sa_layout(a).total + 1024 > kSmemBudget) return false;
    *out = a;
    return true;
}
bool tc_sa_eligible(const psa_mlp* mlp, int c, int nsample, TcArgs* out) {
    TcArgs a3;
    if (!tc_sa_eligible(mlp, c, nsample, &a3, 3)) return false;
    if (g_tc_np == 3) { *out = a3; return true; }
    return tc_sa_eligible(mlp, c, nsample, out, 2);
}

// per tensor layer: an fp16x2 image (when the caller brought none) + the bf16x3 image of the guarded rerun / of mode 2
size_t tc_sa_workspace_bytes(const TcArgs& a, int b, int n, int c) {
    size_t bytes = 256;       // tile counters + range flags
    for (int l = 0; l < a.nl; ++l) bytes += tc_image_alloc_bytes(a.Kd[l], a.Ntot[l], 2) + tc_image_alloc_bytes(a.Kd[l], a.Ntot[l], 3);
    if (c > 0) bytes += (((size_t)b * n * a.C1 * sizeof(float) + 255) & ~(size_t)255) + tc_dense_image_bytes(c, a.C1);
    return bytes;
}

// tile width (with the image-format flag of the current split) of the tensor layers of a level: 64-wide blocks
static int tc_sa_image_nt() { return kSaNt | image_flag(g_tc_np); }

template <int NP, int C1, int NL, int N0>
static int launch_tc_sa_shape(const TcArgs& a, long long ctas_needed, size_t smem, cudaStream_t st) {
    PSA_CUDA(cudaFuncSetAttribute(tc_sa_kernel<NP, C1, NL, N0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // persistent CTAs: as many as are resident at once (two per SM for the smaller levels), never more than there is work for
    int dev = 0, sms = 0, per_sm = 0;
    PSA_CUDA(cudaGetDevice(&dev));
    PSA_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PSA_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tc_sa_kernel<NP, C1, NL, N0>, kSaThreads, smem));
    const long long resident = (long long)sms * (per_sm > 0 ? per_sm : 1);
    const int ctas = (int)(ctas_needed < 1 ? 1 : ctas_needed < resident ? ctas_needed : resident);
    tc_sa_kernel<NP, C1, NL, N0><<<ctas, kSaThreads, smem, st>>>(a);
    return check_launch("tc_sa_kernel");
}

template <int NP>
static int launch_tc_sa_np(TcArgs& a, cudaStream_t st) {
    // chunks of one unit (see tc_sa_kernel): a unit is a warpgroup, or the whole CTA when K = 128 or the last layer streams.
    // The units' pooling buffers sit after the layout, in the shared memory the SM has above the budget tc_sa_eligible checks
    // (4 KB are left for the static arrays).  A level whose warpgroup buffers do not fit keeps joint units, and one whose joint
    // buffer does not fit next to a resident last layer streams that layer: its buffer then holds 64 columns (at most 1 KB),
    // and its layout is no larger than the resident one (a last layer of 64 channels never gets here).
    const uint32_t limit = 223u * 1024u;
    auto fits = [&] { return tc_sa_layout(a).total + 1024u + sa_pool_bytes(a) <= limit; };
    a.joint = a.K == 128 || a.stream_last;
    if (!a.joint && !fits()) a.joint = 1;
    if (!fits()) a.stream_last = 1;
    PSA_REQUIRE(fits(), "sa_module: internal error (pooling buffer does not fit)");
    const int C = sa_chunk(a.K, a.joint);
    const long long nchunks = (a.groups + C - 1) / C;
    const long long ctas_needed = a.joint ? nchunks : (nchunks + 1) / 2;   // two units per CTA
    const size_t smem = (size_t)tc_sa_layout(a).total + 1024 + sa_pool_bytes(a);
    // shapes accepted by tc_sa_eligible: C1 in {64, 128}, one or two tensor layers, an inner layer 64 or 128 wide
    if (a.nl == 1) return a.C1 == 64 ? launch_tc_sa_shape<NP, 64, 1, 0>(a, ctas_needed, smem, st) : launch_tc_sa_shape<NP, 128, 1, 0>(a, ctas_needed, smem, st);
    if (a.C1 == 64) return a.Ntot[0] == 64 ? launch_tc_sa_shape<NP, 64, 2, 64>(a, ctas_needed, smem, st) : launch_tc_sa_shape<NP, 64, 2, 128>(a, ctas_needed, smem, st);
    return a.Ntot[0] == 64 ? launch_tc_sa_shape<NP, 128, 2, 64>(a, ctas_needed, smem, st) : launch_tc_sa_shape<NP, 128, 2, 128>(a, ctas_needed, smem, st);
}

// One set-abstraction level on the SA kernel (`a` = eligibility result for the current split): weight images, the U GEMM
// of the feature part of layer 1, the level, and -- fp16x2 -- its guarded bf16x3 rerun.  w1c: optional centre weights (EdgeConv).
static int tc_sa_run(TcArgs& a, int b, int n, int m, int c, int nsample, const float* xyz, const float* new_xyz, const float* points,
                     const int* idx, const psa_mlp* mlp, const float* w1c, float* out, void* workspace, cudaStream_t st) {
    int rc = PSA_OK;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    unsigned int* region = reinterpret_cast<unsigned int*>(ws);
    const StepWords words = step_words(region, 1);
    PSA_CUDA(cudaMemsetAsync(ws, 0, 256, st));
    ws += 256;
    RingWeights w[kMaxTcLayers];
    for (int l = 0; l < a.nl; ++l) {
        const int K = a.Kd[l], N = a.Ntot[l];
        w[l] = RingWeights{K, K, N, kSaNt, mlp->weight[1 + l], ws, ws + tc_image_alloc_bytes(K, N, 2), prebuilt_image(mlp, 1 + l, 0, tc_sa_image_nt())};
        ws += tc_image_alloc_bytes(K, N, 2) + tc_image_alloc_bytes(K, N, 3);
    }
    const float* uf = nullptr;
    if (c > 0) {
        // V = s (points . W1[3:,:] + xyz . W1[:3,:]) + t  once per source point (rows b*n), no ReLU: the level subtracts the
        // centre's part before it
        const long long rows = (long long)b * n;
        DenseStep u{rows, c, a.C1, 1, 0, points, mlp->weight[0] + (size_t)3 * a.C1, mlp->scale[0], mlp->shift[0], reinterpret_cast<float*>(ws)};
        u.xyz3 = xyz;
        u.w3 = mlp->weight[0];
        u.prebuilt = prebuilt_image(mlp, 0, 3, tc_dense_nt(rows, a.C1));
        u.img = ws + (((size_t)rows * a.C1 * sizeof(float) + 255) & ~(size_t)255);
        u.words = step_words(region, 0);
        if ((rc = run_dense(u, st)) != PSA_OK) return rc;
        uf = u.out;
    }
    auto fill = [&](TcArgs& t) {
        t.groups = (long long)b * m; t.K = nsample; t.n = n; t.m = m;
        t.xyz = xyz; t.new_xyz = new_xyz; t.idx = idx; t.out = out; t.uf = uf;
        t.w1x = mlp->weight[0]; t.s1 = mlp->scale[0]; t.t1 = mlp->shift[0]; t.relu1 = mlp->relu[0];
        t.ovf = nullptr; t.run_if = nullptr; t.w1c = w1c;
        for (int l = 0; l < t.nl; ++l) {
            t.s[l] = mlp->scale[1 + l]; t.t[l] = mlp->shift[1 + l]; t.relu[l] = mlp->relu[1 + l]; t.wflag[l] = nullptr; t.colscale[l] = nullptr;
        }
    };
    fill(a);
    for (int l = 0; l < a.nl; ++l) {
        if ((rc = ring_image(w[l], a.np, nullptr, st, a.image[l])) != PSA_OK) return rc;
        if (a.np == 2) { a.wflag[l] = image_trailer(a.image[l], w[l].Kp, w[l].N); a.colscale[l] = image_colscale(a.image[l], w[l].Kp, w[l].N); }
    }
    a.tile_counter = words.counters;
    if (a.np == 3) return launch_tc_sa_np<3>(a, st);
    a.ovf = words.flag;
    rc = launch_tc_sa_np<2>(a, st);
    if (rc != PSA_OK) return rc;
    // guarded rerun with bf16x3 operands: image builds and the level itself are no-ops unless the fp16x2 pass raised the flag
    TcArgs a3;
    PSA_REQUIRE(tc_sa_eligible(mlp, c, nsample, &a3, 3), "sa_module: internal error (bf16x3 eligibility)");
    fill(a3);
    for (int l = 0; l < a3.nl; ++l)
        if ((rc = ring_image(w[l], 3, words.flag, st, a3.image[l])) != PSA_OK) return rc;
    a3.tile_counter = words.counters + 1;
    a3.run_if = words.flag;
    return launch_tc_sa_np<3>(a3, st);
}

// ------------------------------------------------------------------------------------------------------------------
// tc_group_all_kernel -- a whole three-layer group-all level (pointnet_sa_module(group_all=True) with 128 points per cloud)
// in one launch, fp16x2 operands.  A 128-row tile of tc_dense_kernel is exactly one cloud here, so a thread-block cluster of
// four CTAs owns one cloud and the activations between the layers never leave it:
//   * CTA rank r computes columns [r N_l / 4, (r + 1) N_l / 4) of each layer for all 128 rows: layer 0 (K = c, the xyz rows of
//     W1 as the epilogue side input) and layer 1 in one 64- or 128-column pass each, the last layer in 128-column passes, each
//     followed by the max over the 128 rows -- a plain store of out[cloud, col];
//   * the slices of layers 0 and 1 stay in the CTA's own shared memory, written once after the affine and ReLU as the Split<2>
//     pieces the next layer's wgmma takes, in A-fragment order (ga_frag_off), 32 KB per 64 columns.  K block kb of layer l + 1
//     lives in the CTA that owns those columns of layer l: every consumer thread loads its fragments of it with eight 16-byte
//     loads (ld.shared::cluster when a peer owns it) while block kb - 1's wgmma group runs -- nothing to split, and the loads
//     are not waited for until block kb's group is issued.  Layer 0's input rows are read from global memory and split by the
//     consumers (4 KB of 32-byte sectors per block and warp, from L2: the four CTAs of a cloud read the same rows);
//   * one producer warp streams the weight blocks of all three layers through one ring of 32 KB stages (cp.async.bulk from
//     the layers' fp16x2 images, whatever their tile width), so the next layer's first blocks land during this layer's epilogue.
// Arithmetic is tc_dense_kernel's: per 64-wide K block a fresh wgmma sum over the Split<2> pieces in the same order, added into
// fp32 accumulators in increasing kb, then the same epilogue -- every element is bitwise what the three-launch chain computes.
// Like it, the kernel raises *ovf when a leading piece it stores leaves the fp16 range or a weight image is flagged; the
// launcher queues the chain's bf16x3 reruns behind it, conditional on that word.
// Synchronisation across the cluster (mbarriers only: the producer warps have returned by then and must not be waited for):
//   1. every CTA's barriers are initialised before any peer arrives on them: one cluster barrier of all threads at the start,
//      before any warp returns;
//   2. a layer's slice is complete in every CTA before a peer reads it: the consumers finish their stores, meet on a named
//      barrier, and four threads arrive (release, cluster scope) on s_ready[l] of each of the four CTAs; the consumers of every
//      CTA wait on their own s_ready[l] (acquire, cluster scope) before the next layer's first read;
//   3. no CTA exits while a peer may still read its slices: the same handshake on s_done after the last layer's last read.
//      Slices are written once, so nothing is overwritten while a peer may read it.
// ------------------------------------------------------------------------------------------------------------------
struct TcGroupAllArgs {
    int c;                             // input features (K of layer 0), a multiple of 64
    int N[3];                          // layer widths
    int Nt[3];                         // tile width of each layer's weight image (64 | 128)
    const float* points;               // (b, 128, c), 16-byte aligned
    const float* xyz;                  // (b, 128, 3)
    const float* w3;                   // (3, N[0]): the xyz rows of layer 0's weights
    const uint8_t* image[3];           // fp16x2 weight images (blocks, column factors, trailer)
    const float* colscale[3];
    const unsigned int* wflag[3];
    const float* scale[3];             // or null
    const float* shift[3];             // or null
    int relu[3];
    float* out;                        // (b, N[2])
    unsigned int* ovf;                 // raised when the result is invalid (the bf16x3 reruns then replace it)
};

constexpr int kGaStages = 3;
constexpr uint32_t kGaStageBytes = 32768u;      // one K block of 128 weight columns, two fp16 pieces
constexpr uint32_t kGaSmemBudget = 222u * 1024u;
// A 64-column block of a slice holds the next layer's A fragments of all 128 rows, already split: for consumer warp w, piece
// pc and K step ks (q = 4 pc + ks), lane l's four registers A[pc][ks][0..3] are 16 bytes at ga_frag_off(w, l, q) -- a warp's
// 16-byte loads of one q are 512 contiguous bytes.  Two fp16 pieces of 128 x 64 values: 32 KB.
constexpr uint32_t kGaSliceBytes = 32768u;
__device__ __forceinline__ uint32_t ga_frag_off(int warp, int lane, int q) { return (uint32_t)(((warp * 8 + q) * 32 + lane) * 16); }
// dynamic shared memory: 1 KB alignment, the ring, the slices of layers 0 and 1 (W0 + W1 columns), the affine of every layer
__host__ __device__ inline uint32_t group_all_smem(int W0, int W1, int W2) {
    return 1024u + kGaStages * kGaStageBytes + (uint32_t)(W0 + W1) / 64u * kGaSliceBytes + 12u * (uint32_t)(W0 + W1 + W2);
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r));
    return r;
}
// the shared::cluster address of the same variable in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void ld_cluster_v4(uint32_t addr, uint32_t (&v)[4]) {
    asm volatile("ld.shared::cluster.v4.u32 {%0, %1, %2, %3}, [%4];\n" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ld_shared_v4(uint32_t addr, uint32_t (&v)[4]) {
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];\n" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, const uint32_t (&v)[4]) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};\n" ::"r"(addr), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}
// arrive on the mbarrier at shared::cluster address `addr` (any CTA of the cluster), releasing this thread's prior writes -- and
// those ordered before them by a barrier -- at cluster scope
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t addr) {
    asm volatile("fence.acq_rel.cluster;\n\tmbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];\n" ::"r"(addr) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    const uint32_t addr = smem_u32(bar);
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}\n"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!done);
}

#ifdef PSA_GA_STAMPS
// K-block timeline (tools/group_all_timing.py builds a separate library with -DPSA_GA_STAMPS; libpsa.so has none of this):
// thread 0 of each consumer warpgroup of CTA i < kGaStampCtas writes clock64() at ring use u < kGaStampUses: [0] weight block
// ready, [1] wgmma group issued, [2] the next K block's A operand in registers, [3] group retired; [kGaStampUses - 1][0] is the
// warpgroup's start.
constexpr int kGaStampCtas = 256, kGaStampUses = 64;
__device__ long long g_ga_stamps[kGaStampCtas][2][kGaStampUses][4];
extern "C" PSA_API int psa_group_all_stamps(long long* dst) {
    return cudaMemcpyFromSymbol(dst, g_ga_stamps, sizeof(g_ga_stamps)) == cudaSuccess ? 0 : 1;
}
#define GA_STAMP(u, k)                                                                                              \
    do {                                                                                                            \
        if ((threadIdx.x & 127) == 0 && blockIdx.x < kGaStampCtas && (u) < kGaStampUses)                            \
            g_ga_stamps[blockIdx.x][threadIdx.x >> 7][(u)][(k)] = clock64();                                        \
    } while (0)
// the stamp after a volatile store of a value computed from register r, so the load that wrote r has landed (x * 0 cannot
// be folded away in IEEE arithmetic)
#define GA_STAMP_AFTER(u, k, r)                                                                                     \
    do {                                                                                                            \
        if ((threadIdx.x & 127) == 0 && blockIdx.x < kGaStampCtas && (u) < kGaStampUses) {                          \
            volatile long long* p_ = &g_ga_stamps[blockIdx.x][threadIdx.x >> 7][(u)][(k)];                          \
            *p_ = (long long)__float_as_uint(__fmul_rn(__uint_as_float(r), 0.f));                                   \
            *p_ = clock64();                                                                                        \
        }                                                                                                           \
    } while (0)
#else
#define GA_STAMP(u, k) \
    do {               \
    } while (0)
#define GA_STAMP_AFTER(u, k, r) \
    do {                        \
    } while (0)
#endif

// NC0, NC1: 64-column chunks of the layer-0 and layer-1 slices (one pass each); the last layer runs in 128-column passes
template <int NC0, int NC1>
__global__ void __cluster_dims__(4, 1, 1) __launch_bounds__(kRingThreads, 1)
tc_group_all_kernel(const __grid_constant__ TcGroupAllArgs a) {
    constexpr int NP = 2, S = kGaStages;
    constexpr uint32_t piece = 8192u, chunk = 16384u;               // a 64-column chunk of a stage: its two pieces
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_full[S], s_empty[S], s_ready[2], s_done;
    __shared__ float s_red[8][128];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t rank = cluster_ctarank();
    const int cloud = blockIdx.x >> 2;
    uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    constexpr int W0 = 64 * NC0, W1 = 64 * NC1;                     // slice widths
    const int W2 = a.N[2] / 4;
    uint8_t* slice0 = base + S * kGaStageBytes;
    uint8_t* slice1 = slice0 + NC0 * kGaSliceBytes;
    float* aff0 = reinterpret_cast<float*>(slice1 + NC1 * kGaSliceBytes);   // per layer: scale x column factor, shift, 1 / column factor
    float* aff1 = aff0 + 3 * W0;
    float* aff2 = aff1 + 3 * W1;
    {
        float* aff[3] = {aff0, aff1, aff2};
        const int W[3] = {W0, W1, W2};
#pragma unroll
        for (int l = 0; l < 3; ++l)
            for (int i = tid; i < W[l]; i += kRingThreads) {
                const int col = (int)rank * W[l] + i;
                const float cs = __ldg(a.colscale[l] + col);
                aff[l][i] = (a.scale[l] ? __ldg(a.scale[l] + col) : 1.f) * cs;
                aff[l][W[l] + i] = a.shift[l] ? __ldg(a.shift[l] + col) : 0.f;
                aff[l][2 * W[l] + i] = pow2_rcp(cs);
            }
    }
    if (tid == 0) {
        for (int i = 0; i < S; ++i) { mbar_init(&s_full[i], 1); mbar_init(&s_empty[i], kRingConsumers / 32); }
        mbar_init(&s_ready[0], 4); mbar_init(&s_ready[1], 4); mbar_init(&s_done, 4);
        fence_mbar_init();
    }
    __syncthreads();
    cluster_sync_all();                                             // hazard 1: the peers' barriers are initialised
    const int KC[3] = {a.c / 64, 4 * W0 / 64, 4 * W1 / 64};

    if (warp >= kRingConsumers / 32) {
        // ---- producer: the weight blocks of every pass, in the consumers' order ----
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
        if (warp != kRingConsumers / 32) return;
        uint32_t u = 0;                                             // ring uses
#pragma unroll
        for (int l = 0; l < 3; ++l) {
            const int pw = l == 0 ? W0 : l == 1 ? W1 : 128, passes = l == 2 ? W2 / 128 : 1, Nt = a.Nt[l];
            for (int p = 0; p < passes; ++p) {
                const int j0 = ((int)rank * (l == 0 ? W0 : l == 1 ? W1 : W2) + p * pw) / 64;   // first 64-column chunk of the pass
                for (int kb = 0; kb < KC[l]; ++kb, ++u) {
                    const int s = (int)(u % S);
                    if (u >= (uint32_t)S) mbar_wait(&s_empty[s], ((u / S) - 1u) & 1u);
                    if (lane == 0) {
                        mbar_expect_tx(&s_full[s], (uint32_t)(pw / 64) * chunk);
                        for (int c = 0; c < pw / 64; ++c) {
                            uint8_t* dst = base + (uint32_t)s * kGaStageBytes + (uint32_t)c * chunk;
                            const int j = j0 + c;
                            if (Nt == 64) {                         // block (j, kb) is the chunk, both pieces
                                bulk_g2s(dst, a.image[l] + ((size_t)j * KC[l] + kb) * chunk, chunk, &s_full[s]);
                            } else {                                // half j & 1 of each piece of block (j / 2, kb)
                                const uint8_t* src = a.image[l] + ((size_t)(j >> 1) * KC[l] + kb) * (2u * chunk) + (uint32_t)(j & 1) * piece;
                                bulk_g2s(dst, src, piece, &s_full[s]);
                                bulk_g2s(dst + piece, src + 2u * piece, piece, &s_full[s]);
                            }
                        }
                    }
                }
            }
        }
        return;
    }

    // ---- consumers: warp w holds rows 16w + g and 16w + g + 8 of the cloud ----
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
    const int g = lane >> 2, t = lane & 3;
    const int rl[2] = {warp * 16 + g, warp * 16 + g + 8};
    uint32_t ovf = 0u;
    uint32_t u = 0;                                                 // ring uses
    GA_STAMP(kGaStampUses - 1, 0);

    // one pass of layer L: 64 NC columns starting at column `lc` of this CTA's slice
    auto pass = [&](auto Ltag, auto NCtag, int lc) {
        constexpr int L = decltype(Ltag)::value, NC = decltype(NCtag)::value;
        const int nkb = KC[L];
        // K block kb of the layer's input -> A fragments: layer 0 splits 16 float2 loads from global memory, layers 1 and 2 load
        // the pieces the owner of the block stored (8 16-byte loads, nothing to wait for until the block's wgmma group)
        auto prep = [&](uint32_t (&A)[NP][4][4], int kb) {
            if constexpr (L == 0) {
                const float* xb = a.points + (size_t)cloud * 128 * a.c + kb * 64;
#pragma unroll
                for (int s = 0; s < 4; ++s)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const float2 x = __ldg(reinterpret_cast<const float2*>(xb + (size_t)rl[i] * a.c + 16 * s + 8 * h + 2 * t));
                            put_a<NP, 4>(A, s, i + 2 * h, x.x, x.y, ovf);
                        }
            } else {
                constexpr int Wp = L == 1 ? W0 : W1;                // the input's slice width: block kb is in CTA kb * 64 / Wp
                const uint32_t owner = (uint32_t)(kb * 64 / Wp);
                const uint32_t src = smem_u32(L == 1 ? slice0 : slice1) + (uint32_t)((kb * 64) % Wp / 64) * kGaSliceBytes + ga_frag_off(warp, lane, 0);
                if (owner == rank) {
#pragma unroll
                    for (int q = 0; q < NP * 4; ++q) ld_shared_v4(src + (uint32_t)q * 512u, A[q >> 2][q & 3]);
                } else {
                    const uint32_t rsrc = mapa_shared(src, owner);
#pragma unroll
                    for (int q = 0; q < NP * 4; ++q) ld_cluster_v4(rsrc + (uint32_t)q * 512u, A[q >> 2][q & 3]);
                }
            }
        };
        float acc[NC][32];
        // block kb (ring use u): issue its group on A, prepare block kb + 1 into An while it runs, wait, release the stage, add
        auto step = [&](const uint32_t (&A)[NP][4][4], uint32_t (&An)[NP][4][4], int kb) {
            const int s = (int)(u % S);
            mbar_wait(&s_full[s], (u / S) & 1u);
            GA_STAMP(u, 0);
            const uint32_t wb = smem_u32(base) + (uint32_t)s * kGaStageBytes;
            float d[NC][32];
            wg_fence();
#pragma unroll
            for (int tt = 0; tt < Split<NP>::kTerms; ++tt)
#pragma unroll
                for (int ks = 0; ks < 4; ++ks)
#pragma unroll
                    for (int c = 0; c < NC; ++c)
                        wg_mma_rs<NP>(d[c], A[Split<NP>::a(tt)][ks][0], A[Split<NP>::a(tt)][ks][1], A[Split<NP>::a(tt)][ks][2], A[Split<NP>::a(tt)][ks][3],
                                      wg_desc(wb + (uint32_t)c * chunk + Split<NP>::w(tt) * piece + (uint32_t)ks * 32u), (tt | ks) ? 1u : 0u);
            wg_commit();
            GA_STAMP(u, 1);
            if (kb + 1 < nkb) prep(An, kb + 1);
            GA_STAMP_AFTER(u, 2, An[1][3][3]);
            wg_wait_all();
            GA_STAMP(u, 3);
            __syncwarp();
            if (lane == 0) mbar_arrive1(&s_empty[s]);               // weights consumed: the stage may be refilled
            ++u;
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                wg_fence_acc(d[c]);
#pragma unroll
                for (int e = 0; e < 32; ++e) acc[c][e] = kb ? acc[c][e] + d[c][e] : d[c][e];
            }
        };
        {
            uint32_t A0[NP][4][4], A1[NP][4][4];
            prep(A0, 0);
            for (int kb = 0;; kb += 2) {
                step(A0, A1, kb);
                if (kb + 1 == nkb) break;
                step(A1, A0, kb + 1);
                if (kb + 2 == nkb) break;
            }
        }

        // ---- epilogue: tc_dense_kernel's, in the fragment layout ----
        constexpr int W = L == 0 ? W0 : L == 1 ? W1 : 0;
        const int Wl = L == 2 ? W2 : W;
        const float* aff = L == 0 ? aff0 : L == 1 ? aff1 : aff2;
        float xs[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
        if constexpr (L == 0)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int k = 0; k < 3; ++k) xs[i][k] = __ldg(a.xyz + ((size_t)cloud * 128 + rl[i]) * 3 + k);
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            uint32_t fr[NP][4];                                     // L < 2: the A fragments of K step j / 2 of the next layer
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int cl = c * 64 + 8 * j + 2 * t, ls = lc + cl;   // column in the pass, in the slice
                float y[2][2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float sc = aff[ls + e], sh = aff[Wl + ls + e];
                    float w0 = 0.f, w1 = 0.f, w2 = 0.f;
                    if constexpr (L == 0) {
                        const int col = (int)rank * W0 + ls + e;
                        const float f = aff[2 * Wl + ls + e];
                        w0 = __ldg(a.w3 + col) * f; w1 = __ldg(a.w3 + a.N[0] + col) * f; w2 = __ldg(a.w3 + 2 * a.N[0] + col) * f;
                    }
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        float x = acc[c][4 * j + 2 * i + e];
                        if constexpr (L == 0) x = fmaf(xs[i][2], w2, fmaf(xs[i][1], w1, fmaf(xs[i][0], w0, x)));
                        x = fmaf(x, sc, sh);
                        if (a.relu[L]) x = fmaxf(x, 0.f);
                        y[i][e] = x;
                    }
                }
                if constexpr (L < 2) {
                    // the pieces the next layer's wgmma takes (the split its readers did before, once here, range tracked)
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        uint32_t p[NP];
                        split_pair<NP>(y[i][0], y[i][1], p, ovf);
#pragma unroll
                        for (int pc = 0; pc < NP; ++pc) fr[pc][i + 2 * (j & 1)] = p[pc];
                    }
                    if (j & 1) {
                        const uint32_t sl = smem_u32(L == 0 ? slice0 : slice1) + (uint32_t)c * kGaSliceBytes;
#pragma unroll
                        for (int pc = 0; pc < NP; ++pc) st_shared_v4(sl + ga_frag_off(warp, lane, 4 * pc + (j >> 1)), fr[pc]);
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float m = warp_rowmax16(y[0][e], y[1][e]);
                        if (g == 0) s_red[warp][cl + e] = m;
                    }
                }
            }
        }
        unit_bar_sync(1, kRingConsumers);
        if constexpr (L < 2) {
            // hazard 2: the slice is complete in this CTA -> tell every CTA of the cluster, then wait until all four are
            if (tid < 4) mbar_arrive_cluster(mapa_shared(smem_u32(&s_ready[L]), (uint32_t)tid));
            mbar_wait_cluster(&s_ready[L], 0);
        } else {
            for (int cl = tid; cl < 64 * NC; cl += kRingConsumers) {
                float mx = s_red[0][cl];
                for (int w = 1; w < 8; ++w) mx = fmaxf(mx, s_red[w][cl]);
                a.out[(size_t)cloud * a.N[2] + (size_t)rank * W2 + lc + cl] = mx;
            }
            unit_bar_sync(1, kRingConsumers);                      // s_red is rewritten by the next pass
        }
    };
    pass(std::integral_constant<int, 0>{}, std::integral_constant<int, NC0>{}, 0);
    pass(std::integral_constant<int, 1>{}, std::integral_constant<int, NC1>{}, 0);
    for (int lc = 0; lc < W2; lc += 128) pass(std::integral_constant<int, 2>{}, std::integral_constant<int, 2>{}, lc);

    // hazard 3: the last reads of the peers' slices are done (their values are in the wgmma groups retired above)
    if (tid < 4) mbar_arrive_cluster(mapa_shared(smem_u32(&s_done), (uint32_t)tid));
    if (f16x2_overflowed(ovf) || (tid == 0 && (*a.wflag[0] | *a.wflag[1] | *a.wflag[2]) != 0u)) atomicOr(a.ovf, 1u);
    mbar_wait_cluster(&s_done, 0);
}

// Can this group-all level run as one tc_group_all_kernel launch?  fp16x2 mode, three layers, 128 points per cloud, c a multiple
// of 64 with 16-byte-aligned rows, layer widths N0, N1 in {256, 512} (not both 512: the two slices and the ring must fit in
// shared memory) and N2 a multiple of 512, and a cluster of four such CTAs must fit on the device.  Returns the kernel's
// shared memory, 0 when not eligible.
template <int NC0, int NC1>
static size_t group_all_fits(const psa_mlp* mlp) {
    const size_t smem = group_all_smem(64 * NC0, 64 * NC1, mlp->channels[3] / 4);
    if (smem > kGaSmemBudget) return 0;
    if (cudaFuncSetAttribute(tc_group_all_kernel<NC0, NC1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return 0;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(4, 1, 1);
    cfg.blockDim = dim3(kRingThreads, 1, 1);
    cfg.dynamicSmemBytes = smem;
    int clusters = 0;
    if (cudaOccupancyMaxActiveClusters(&clusters, tc_group_all_kernel<NC0, NC1>, &cfg) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
    return clusters > 0 ? smem : 0;
}
static size_t group_all_eligible(int n, int c, const float* points, const psa_mlp* mlp) {
    if (g_tc_np != 2 || mlp->n_layers != 3 || n != 128 || c < 64 || c % 64 != 0 || (reinterpret_cast<uintptr_t>(points) & 15) != 0) return 0;
    const int N0 = mlp->channels[1], N1 = mlp->channels[2], N2 = mlp->channels[3];
    if (N2 % 512 != 0) return 0;
    if (N0 == 256 && N1 == 256) return group_all_fits<1, 1>(mlp);
    if (N0 == 256 && N1 == 512) return group_all_fits<1, 2>(mlp);
    if (N0 == 512 && N1 == 256) return group_all_fits<2, 1>(mlp);
    return 0;
}

// A chain of inference dense layers (psa_shared_mlp, psa_shared_mlp_grouped, psa_sa_group_all_infer) and its workspace, the one
// layout both the size queries and the launchers read: activations ping-pong between two halves, one image slot per layer,
// fc_small's partial sums when rows <= 32, the zeroed word region last.  Group-all's first layer (row0 = 3) is the K0 = c
// feature rows of its W, the xyz rows the side input.
struct ChainPlan {
    long long rows;
    int L, row0;
    int K[PSA_MAX_MLP_LAYERS], N[PSA_MAX_MLP_LAYERS];
    size_t half, img[PSA_MAX_MLP_LAYERS], fc, words, bytes;   // byte offsets into the workspace; its size
};
static ChainPlan chain_plan(long long rows, const psa_mlp* mlp, int K0, int row0) {
    ChainPlan p{};
    p.rows = rows; p.L = mlp->n_layers; p.row0 = row0;
    int cmax = 0;
    for (int l = 0; l < p.L; ++l) {
        p.K[l] = l == 0 ? K0 : mlp->channels[l];
        p.N[l] = mlp->channels[l + 1];
        if (l > 0) cmax = std::max(cmax, p.K[l]);
    }
    p.half = p.L > 1 ? al256((size_t)rows * cmax * sizeof(float)) : 0;
    size_t off = 2 * p.half, fc = 0;
    for (int l = 0; l < p.L; ++l) {
        p.img[l] = off;
        off += tc_dense_image_bytes(p.K[l], std::max(p.N[l], 64));
        if (rows <= 32) fc = std::max(fc, fc_small_workspace_bytes(p.K[l], p.N[l]));
    }
    p.fc = off;
    p.words = off + al256(fc);
    p.bytes = p.words + 256;
    return p;
}

// layer l of chain p in the workspace ws: x is the first layer's input, xyz group-all's side input, out the last layer's output,
// pool_k the last layer's
static DenseStep chain_step(const ChainPlan& p, int l, int pool_k, const psa_mlp* mlp, const float* x, const float* xyz, float* out, uint8_t* ws) {
    float* half[2] = {reinterpret_cast<float*>(ws), reinterpret_cast<float*>(ws + p.half)};
    const int row0 = l == 0 ? p.row0 : 0;
    DenseStep s{p.rows, p.K[l], p.N[l], l == p.L - 1 ? pool_k : 1, mlp->relu[l], l == 0 ? x : half[(l - 1) & 1],
                mlp->weight[l] + (size_t)row0 * p.N[l], mlp->scale[l], mlp->shift[l], l == p.L - 1 ? out : half[l & 1]};
    if (row0 != 0) { s.xyz3 = xyz; s.w3 = mlp->weight[0]; }
    s.prebuilt = prebuilt_image(mlp, l, row0, tc_dense_nt(p.rows, s.N));
    s.img = ws + p.img[l];
    s.words = step_words(reinterpret_cast<unsigned int*>(ws + p.words), l);
    if (p.rows <= 32) s.fc_partial = reinterpret_cast<float*>(ws + p.fc);
    return s;
}

static int run_chain(const ChainPlan& p, int pool_k, const psa_mlp* mlp, const float* x, const float* xyz, const float* group_add,
                     long long group_rows, float* out, uint8_t* ws, cudaStream_t st) {
    for (int l = 0; l < p.L; ++l) {
        DenseStep s = chain_step(p, l, pool_k, mlp, x, xyz, out, ws);
        s.group_add = l == 0 ? group_add : nullptr;
        s.group_rows = group_rows;
        const int rc = run_dense(s, st);
        if (rc != PSA_OK) return rc;
    }
    return PSA_OK;
}

// The group-all level of psa_sa_group_all_infer on tc_group_all_kernel (group_all_eligible said yes, `smem`), then the bf16x3
// reruns of chain p's three layers, conditional on the kernel's range flag: the output is then what psa_set_mlp_mode(2) gives.
// The layers, their images and the reruns' workspace and tile counters are those of the chain.
static int sa_group_all_cluster(const ChainPlan& p, const float* xyz, const float* points, const psa_mlp* mlp, float* out, uint8_t* ws,
                                size_t smem, cudaStream_t st) {
    unsigned int* flag = step_words(reinterpret_cast<unsigned int*>(ws + p.words), kClusterFlagStep).flag;
    TcGroupAllArgs g{};
    g.c = p.K[0]; g.points = points; g.xyz = xyz; g.w3 = mlp->weight[0]; g.out = out; g.ovf = flag;
    DenseStep s[3];
    int rc;
    for (int l = 0; l < 3; ++l) {
        s[l] = chain_step(p, l, 128, mlp, points, xyz, out, ws);
        const RingWeights w = tc_dense_weights(s[l]);
        if ((rc = ring_image(w, 2, nullptr, st, g.image[l])) != PSA_OK) return rc;
        g.N[l] = w.N; g.Nt[l] = w.Nt;
        g.colscale[l] = image_colscale(g.image[l], w.Kp, w.N); g.wflag[l] = image_trailer(g.image[l], w.Kp, w.N);
        g.scale[l] = s[l].scale; g.shift[l] = s[l].shift; g.relu[l] = s[l].relu;
    }
    const unsigned grid = 4u * (unsigned)(p.rows / 128);
    if (g.N[0] == 256 && g.N[1] == 256) tc_group_all_kernel<1, 1><<<grid, kRingThreads, smem, st>>>(g);
    else if (g.N[0] == 256) tc_group_all_kernel<1, 2><<<grid, kRingThreads, smem, st>>>(g);
    else tc_group_all_kernel<2, 1><<<grid, kRingThreads, smem, st>>>(g);
    if ((rc = check_launch("tc_group_all_kernel")) != PSA_OK) return rc;
    for (int l = 0; l < 3; ++l) {
        const RingWeights w = tc_dense_weights(s[l]);
        rc = ring_rerun(kDenseRing, tc_dense_args(s[l]), tc_dense_units(p.rows, w.N, w.Nt), w, flag, s[l].words.counters + 1, st);
        if (rc != PSA_OK) return rc;
    }
    return PSA_OK;
}

}  // namespace psa

using namespace psa;

extern "C" PSA_API int psa_set_mlp_mode(int mode) {
    PSA_REQUIRE(mode == 0 || mode == 1 || mode == 2,
                "set_mlp_mode: mode must be 0 (tensor cores, fp16x2 operands with the range guard), 1 (fp32 FMA kernels only) or 2 (tensor cores, bf16x3)");
    g_mlp_mode = mode;
    g_tc_np = mode == 2 ? 3 : 2;
    return PSA_OK;
}
extern "C" PSA_API int psa_get_mlp_mode(void) { return g_mlp_mode; }

extern "C" size_t psa_sa_module_workspace_bytes(int b, int n, int m, int c, int nsample, const psa_mlp* mlp) {
    (void)m;
    TcArgs a;
    if (g_mlp_mode != 1 && mlp != nullptr && tc_sa_eligible(mlp, c, nsample, &a)) return tc_sa_workspace_bytes(a, b, n, c);
    return 0;
}

extern "C" int psa_sa_module_infer(int b, int n, int m, int c, float radius, int nsample, const float* xyz,
                                   const float* new_xyz, const float* points, const int* idx_in, const psa_mlp* mlp,
                                   float* out, int* idx_out, int* pts_cnt, void* workspace, size_t workspace_bytes,
                                   psa_stream_t stream) {
    int rc = validate_mlp_public(mlp, "sa_module");
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(b >= 0 && n >= 1 && m >= 0 && c >= 0 && nsample >= 1, "sa_module: bad dims b=%d n=%d m=%d c=%d nsample=%d", b, n, m, c, nsample);
    PSA_REQUIRE(mlp->channels[0] == 3 + c, "sa_module: mlp input width %d != 3 + c (%d)", mlp->channels[0], 3 + c);
    if (b == 0 || m == 0) return PSA_OK;
    PSA_REQUIRE(xyz && new_xyz && out && (points || c == 0), "sa_module: null buffer");
    const int* idx = idx_in;
    if (idx == nullptr) {
        PSA_REQUIRE(idx_out != nullptr, "sa_module: idx_out must be provided when idx_in is NULL (it receives the ball query)");
        rc = psa_query_ball_point(b, n, m, radius, nsample, xyz, new_xyz, idx_out, pts_cnt, stream);
        if (rc != PSA_OK) return rc;
        idx = idx_out;
    }
    cudaStream_t st = as_stream(stream);
    TcArgs a;
    if (g_mlp_mode != 1 && tc_sa_eligible(mlp, c, nsample, &a)) {
        const size_t need = tc_sa_workspace_bytes(a, b, n, c);
        PSA_REQUIRE(workspace != nullptr && workspace_bytes >= need,
                    "sa_module: workspace of %zu bytes required (psa_sa_module_workspace_bytes), got %zu", need, workspace_bytes);
        PSA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "sa_module: workspace must be 256-byte aligned");
        return tc_sa_run(a, b, n, m, c, nsample, xyz, new_xyz, points, idx, mlp, nullptr, out, workspace, st);
    }
    return sa_module_simt(b, n, m, c, nsample, xyz, new_xyz, points, idx, mlp, out, st);
}

extern "C" size_t psa_shared_mlp_workspace_bytes(long long rows, const psa_mlp* mlp) {
    if (mlp == nullptr || mlp->n_layers < 1 || mlp->n_layers > PSA_MAX_MLP_LAYERS) return 0;
    return chain_plan(rows, mlp, mlp->channels[0], 0).bytes;
}

// The layer chain of psa_shared_mlp and psa_shared_mlp_grouped (arguments validated by the caller; group_add: layer 0's per-group input,
// or null).
static int shared_mlp_chain(long long rows, int pool_k, const float* x, const psa_mlp* mlp, const float* group_add, long long group_rows,
                            float* out, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    const ChainPlan p = chain_plan(rows, mlp, mlp->channels[0], 0);
    PSA_REQUIRE(workspace != nullptr && workspace_bytes >= p.bytes, "shared_mlp: workspace of %zu bytes required (got %zu)", p.bytes, workspace_bytes);
    PSA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "shared_mlp: workspace must be 256-byte aligned");
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    cudaStream_t st = as_stream(stream);
    PSA_CUDA(cudaMemsetAsync(ws + p.words, 0, 256, st));
    return run_chain(p, pool_k, mlp, x, nullptr, group_add, group_rows, out, ws, st);
}

extern "C" int psa_shared_mlp(long long rows, int pool_k, const float* x, const psa_mlp* mlp, float* out,
                              void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = validate_mlp_public(mlp, "shared_mlp");
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(rows >= 0 && pool_k >= 1, "shared_mlp: rows=%lld pool_k=%d", rows, pool_k);
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(rows % pool_k == 0, "shared_mlp: rows=%lld is not a multiple of pool_k=%d", rows, pool_k);
    PSA_REQUIRE(x && out, "shared_mlp: null buffer");
    return shared_mlp_chain(rows, pool_k, x, mlp, nullptr, 0, out, workspace, workspace_bytes, stream);
}

extern "C" int psa_shared_mlp_grouped(long long rows, long long group_rows, const float* x, const psa_mlp* mlp, const float* group_add,
                                      float* out, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = validate_mlp_public(mlp, "shared_mlp_grouped");
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(rows >= 0 && group_rows >= 1, "shared_mlp_grouped: rows=%lld group_rows=%lld", rows, group_rows);
    PSA_REQUIRE(rows % group_rows == 0, "shared_mlp_grouped: group_rows=%lld does not divide rows=%lld", group_rows, rows);
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(x && group_add && out, "shared_mlp_grouped: null buffer");
    return shared_mlp_chain(rows, 1, x, mlp, group_add, group_rows, out, workspace, workspace_bytes, stream);
}

// pointnet_sa_module(group_all=True) (pointnet_util.py:59-84,113-127): rows = [xyz, points] (xyz first), MLP, max over the
// n points of each cloud -- without building the (b,n,3+c) concatenation: the feature part [3:,:] of the first layer runs
// as an aligned K = c GEMM on the tensor cores, the three xyz rows of W1 are folded into its epilogue.
extern "C" size_t psa_sa_group_all_workspace_bytes(int b, int n, int c, const psa_mlp* mlp) {
    if (mlp == nullptr || mlp->n_layers < 1 || mlp->n_layers > PSA_MAX_MLP_LAYERS) return 0;
    return chain_plan((long long)b * n, mlp, c, 3).bytes;
}

extern "C" int psa_sa_group_all_infer(int b, int n, int c, const float* xyz, const float* points, const psa_mlp* mlp,
                                      float* out, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = validate_mlp_public(mlp, "sa_group_all");
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(b >= 0 && n >= 1 && c >= 1, "sa_group_all: bad dims b=%d n=%d c=%d", b, n, c);
    PSA_REQUIRE(mlp->channels[0] == 3 + c, "sa_group_all: mlp input width %d != 3 + c (%d)", mlp->channels[0], 3 + c);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(xyz && points && out, "sa_group_all: null buffer");
    const ChainPlan p = chain_plan((long long)b * n, mlp, c, 3);
    PSA_SUPPORTED(dense_on_tc(p.rows, c, p.N[0], p.L == 1 ? n : 1),
                  "sa_group_all: first layer (%d -> %d over %lld rows) is not eligible for the tensor-core path; concatenate and use shared_mlp", c, p.N[0], p.rows);
    PSA_REQUIRE(workspace != nullptr && workspace_bytes >= p.bytes, "sa_group_all: workspace of %zu bytes required (got %zu)", p.bytes, workspace_bytes);
    PSA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "sa_group_all: workspace must be 256-byte aligned");
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    cudaStream_t st = as_stream(stream);
    PSA_CUDA(cudaMemsetAsync(ws + p.words, 0, 256, st));
    // one cluster of four CTAs per cloud when the level allows it; otherwise one launch per layer
    if (g_mlp_mode == 0) {
        const size_t smem = group_all_eligible(n, c, points, mlp);
        if (smem != 0) return sa_group_all_cluster(p, xyz, points, mlp, out, ws, smem, st);
    }
    return run_chain(p, n, mlp, points, xyz, nullptr, 0, out, ws, st);
}

// ------------------------------------------------------------------------------------------------------------------
// EdgeConv, single layer (dgcnn/models/dgcnn.py:41-47 etc.):  max_j relu(BN(W . [x_i ; x_j - x_i] + b)).
//   W . [x_i ; x_j - x_i] = (W_a - W_b) . x_i + W_b . x_j   and, per channel, relu(s*(A_i + B_j) + t) is monotone in B_j
//   (increasing if s >= 0, decreasing otherwise), so the max over the k edges only needs max_j / min_j of B:
//   one (B*N) x C x 2C_out GEMM over POINTS (k-fold fewer rows than the reference's conv over B*N*k edges, tensor cores)
//   + one gather-max pass.  No (B,N,k,2C) edge tensor, no (B,N,k,C_out) activation tensor.
// ------------------------------------------------------------------------------------------------------------------
__global__ void edge_wc_kernel(int c, int N, const float* __restrict__ W, float* __restrict__ Wc) {
    const int total = c * 2 * N;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
        const int kk = e / (2 * N), j = e - kk * 2 * N;
        Wc[e] = j < N ? __ldg(W + (size_t)kk * N + j) - __ldg(W + (size_t)(c + kk) * N + j) : __ldg(W + (size_t)(c + kk) * N + j - N);
    }
}

template <int VEC>   // channels per lane: N = 32 * VEC
__global__ void __launch_bounds__(256)
edge_gather_max_kernel(long long points, int n, int k, int N, const float* __restrict__ AB, const int* __restrict__ nn_idx,
                       const float* __restrict__ scale, const float* __restrict__ shift, int relu, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long warp0 = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    float sc[VEC], sh[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
        sc[v] = scale ? __ldg(scale + lane * VEC + v) : 1.f;
        sh[v] = shift ? __ldg(shift + lane * VEC + v) : 0.f;
    }
    for (long long p = warp0; p < points; p += (long long)gridDim.x * 8) {
        const long long base = (p / n) * n;
        const float* arow = AB + (size_t)p * 2 * N + lane * VEC;
        float a[VEC], mx[VEC], mn[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) { a[v] = __ldg(arow + v); mx[v] = -FLT_MAX; mn[v] = FLT_MAX; }
        const int myj = lane < k ? __ldg(nn_idx + p * k + lane) : 0;          // k <= 32
        for (int j = 0; j < k; ++j) {
            const int nb = __shfl_sync(0xffffffffu, myj, j);
            const float* brow = AB + (size_t)(base + nb) * 2 * N + N + lane * VEC;
#pragma unroll
            for (int v = 0; v < VEC; ++v) { const float bv = __ldg(brow + v); mx[v] = fmaxf(mx[v], bv); mn[v] = fminf(mn[v], bv); }
        }
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
            float y = fmaf(a[v] + (sc[v] >= 0.f ? mx[v] : mn[v]), sc[v], sh[v]);
            if (relu) y = fmaxf(y, 0.f);
            out[(size_t)p * N + lane * VEC + v] = y;
        }
    }
}

static bool edgeconv_algebra_ok(long long rows, int c, int k, const psa_mlp* mlp) {
    const int N = mlp->channels[1];
    return g_mlp_mode != 1 && mlp->n_layers == 1 && rows >= 128 && k <= 32 && (N == 32 || N == 64 || N == 128 || N == 256) && c >= 1;
}

// Multi-layer EdgeConv over 3-D points (DGCNN's input transform net, dgcnn/models/transform_nets.py:13-27: [x_i, x_j - x_i] ->
// 64 -> 128 -> max over k) on the set-abstraction kernel: W1 . [x_i ; x_j - x_i] = W1[0:3] . x_i + W1[3:6] . (x_j - x_i) is exactly
// a level whose centres are the points themselves, with W1[3:6] as the xyz weights and W1[0:3] as centre weights (TcArgs::w1c); the
// k <= 32 neighbours are padded to the kernel's 32-row neighbourhoods by repeating the first one (a max-pool ignores duplicates).
__global__ void edge_pad_idx_kernel(long long rows, int k, const int* __restrict__ idx, int* __restrict__ idx32) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < rows * 32; e += (long long)gridDim.x * blockDim.x) {
        const long long r = e >> 5;
        const int j = (int)(e & 31);
        idx32[e] = __ldg(idx + r * k + (j < k ? j : 0));
    }
}
static bool edgeconv_dual_ok(int c, int k, const psa_mlp* mlp, psa_mlp* m2, TcArgs* a) {
    if (g_mlp_mode == 1 || c != 3 || k < 1 || k > 32 || mlp->n_layers < 2) return false;
    *m2 = *mlp;
    m2->channels[0] = 3;
    m2->weight[0] = mlp->weight[0] + (size_t)3 * mlp->channels[1];
    for (int l = 0; l < PSA_MAX_MLP_LAYERS; ++l) { m2->image[l] = nullptr; m2->image_nt[l] = 0; m2->image_row0[l] = 0; }
    return tc_sa_eligible(m2, 0, 32, a);
}

// The path of a single-layer EdgeConv call and its workspace, read by both psa_edgeconv_workspace_bytes and psa_edgeconv_infer.
// Dual: the padded neighbour indices, then tc_sa_run's workspace at `off`.  Algebra: Wc, AB at `off`, the GEMM's image slot at
// `img`, the zeroed word region at `words`.  FMA (the fused kernel): none.
struct EdgePlan {
    enum Path { kFma, kDual, kAlgebra } path = kFma;
    psa_mlp m2;                       // dual: the level's MLP and its eligibility result
    TcArgs a;
    size_t off = 0, img = 0, words = 0, bytes = 0;
};
static EdgePlan edgeconv_plan(int b, int n, int c, int k, const psa_mlp* mlp) {
    EdgePlan p;
    const long long rows = (long long)b * n;
    if (edgeconv_dual_ok(c, k, mlp, &p.m2, &p.a)) {
        p.path = EdgePlan::kDual;
        p.off = al256((size_t)rows * 32 * 4);
        p.bytes = p.off + tc_sa_workspace_bytes(p.a, b, n, 0);
    } else if (edgeconv_algebra_ok(rows, c, k, mlp)) {
        const int N = mlp->channels[1];
        p.path = EdgePlan::kAlgebra;
        p.off = al256((size_t)c * 2 * N * 4);
        p.img = p.off + al256((size_t)rows * 2 * N * 4);
        p.words = p.img + tc_dense_image_bytes(c, 2 * N);
        p.bytes = p.words + 256;
    }
    return p;
}

extern "C" size_t psa_edgeconv_workspace_bytes(int b, int n, int c, int k, const psa_mlp* mlp) {
    return mlp == nullptr ? 0 : edgeconv_plan(b, n, c, k, mlp).bytes;
}

extern "C" int psa_edgeconv_infer(int b, int n, int c, int k, const float* x, const int* nn_idx, const psa_mlp* mlp,
                                  float* out, void* workspace, size_t workspace_bytes, psa_stream_t stream) {
    int rc = validate_mlp_public(mlp, "edgeconv");
    if (rc != PSA_OK) return rc;
    PSA_REQUIRE(b >= 0 && n >= 0 && c >= 1 && k >= 1, "edgeconv: bad dims b=%d n=%d c=%d k=%d", b, n, c, k);
    PSA_REQUIRE(mlp->channels[0] == 2 * c, "edgeconv: mlp input width %d != 2*c (%d)", mlp->channels[0], 2 * c);
    if (b == 0 || n == 0) return PSA_OK;
    PSA_REQUIRE(x && nn_idx && out, "edgeconv: null buffer");
    cudaStream_t st = as_stream(stream);
    const long long rows = (long long)b * n;
    EdgePlan p = edgeconv_plan(b, n, c, k, mlp);
    if (p.path == EdgePlan::kFma) return edgeconv_simt(b, n, c, k, x, nn_idx, mlp, out, st);
    PSA_REQUIRE(workspace != nullptr && workspace_bytes >= p.bytes, "edgeconv: workspace of %zu bytes required (got %zu)", p.bytes, workspace_bytes);
    PSA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "edgeconv: workspace must be 256-byte aligned");
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    if (p.path == EdgePlan::kDual) {
        int* idx32 = reinterpret_cast<int*>(ws);
        edge_pad_idx_kernel<<<(unsigned)((rows * 32 + 255) / 256 < 65535 * 4 ? (rows * 32 + 255) / 256 : 65535 * 4), 256, 0, st>>>(rows, k, nn_idx, idx32);
        rc = check_launch("edge_pad_idx_kernel");
        if (rc != PSA_OK) return rc;
        return tc_sa_run(p.a, b, n, n, 0, 32, x, x, nullptr, idx32, &p.m2, mlp->weight[0], out, ws + p.off, st);
    }
    const int N = mlp->channels[1];
    float* Wc = reinterpret_cast<float*>(ws);
    edge_wc_kernel<<<(c * 2 * N + 255) / 256, 256, 0, st>>>(c, N, mlp->weight[0], Wc);
    DenseStep ab{rows, c, 2 * N, 1, 0, x, Wc, nullptr, nullptr, reinterpret_cast<float*>(ws + p.off)};
    ab.img = ws + p.img;
    ab.words = step_words(reinterpret_cast<unsigned int*>(ws + p.words), 0);
    if (dense_on_tc(rows, c, 2 * N, 1)) PSA_CUDA(cudaMemsetAsync(ws + p.words, 0, 256, st));
    if ((rc = run_dense(ab, st)) != PSA_OK) return rc;
    const int grid = (int)((rows + 7) / 8 < (long long)kNumSMs * 8 ? (rows + 7) / 8 : (long long)kNumSMs * 8);
    const int vec = N / 32;
#define PSA_EDGE_LAUNCH(V) edge_gather_max_kernel<V><<<grid, 256, 0, st>>>(rows, n, k, N, ab.out, nn_idx, mlp->scale[0], mlp->shift[0], mlp->relu[0], out)
    if (vec == 1) PSA_EDGE_LAUNCH(1); else if (vec == 2) PSA_EDGE_LAUNCH(2); else if (vec == 4) PSA_EDGE_LAUNCH(4); else PSA_EDGE_LAUNCH(8);
#undef PSA_EDGE_LAUNCH
    return check_launch("edge_gather_max_kernel");
}

extern "C" int psa_prepare_weight_image(int K, int N, int row0, int nt, const float* W, void* image, psa_stream_t stream) {
    const int ntw = nt & ~kImageFlags;        // nt as returned by psa_mlp_image_plan: tile width | format flag
    PSA_REQUIRE((nt & kImageFlags) == kImageBf16x3 || (nt & kImageFlags) == kImageF16x2, "prepare_weight_image: nt=%d carries no image format flag", nt);
    PSA_REQUIRE(K >= 1 && N >= 64 && N % 64 == 0 && row0 >= 0 && row0 < K && (ntw == 64 || ntw == 128) && N % ntw == 0,
                "prepare_weight_image: bad arguments K=%d N=%d row0=%d nt=%d", K, N, row0, nt);
    PSA_REQUIRE(W && image, "prepare_weight_image: null buffer");
    const int Ki = K - row0, Kp = (Ki + 63) & ~63;
    int rc = build_image(Ki, Kp, N, nt, W + (size_t)row0 * N, reinterpret_cast<uint8_t*>(image), as_stream(stream));
    if (rc != PSA_OK || (nt & kImageF16x2) == 0) return rc;
    // fp16x2 images carry the bf16x3 image of the range guard's rerun right behind them
    return build_image(Ki, Kp, N, ntw | kImageBf16x3, W + (size_t)row0 * N, reinterpret_cast<uint8_t*>(image) + tc_image_alloc_bytes(Kp, N, 2), as_stream(stream));
}

extern "C" int psa_mlp_image_plan(int usage, long long rows, int pool_k, int c, int nsample, const psa_mlp* mlp,
                                  int nt[PSA_MAX_MLP_LAYERS], int row0[PSA_MAX_MLP_LAYERS], size_t bytes[PSA_MAX_MLP_LAYERS]) {
    int rc = validate_mlp_public(mlp, "mlp_image_plan");
    if (rc != PSA_OK) return rc;
    for (int l = 0; l < PSA_MAX_MLP_LAYERS; ++l) { nt[l] = 0; row0[l] = 0; bytes[l] = 0; }
    if (g_mlp_mode == 1) return PSA_OK;
    if (usage == PSA_USAGE_SHARED_MLP || usage == PSA_USAGE_SA_GROUP_ALL) {
        const int r0 = usage == PSA_USAGE_SA_GROUP_ALL ? 3 : 0;
        const ChainPlan p = chain_plan(rows, mlp, mlp->channels[0] - r0, r0);
        for (int l = 0; l < p.L; ++l) {
            const int K = p.K[l], N = p.N[l];
            if (dense_on_tc(rows, K, N, l == p.L - 1 ? pool_k : 1)) { nt[l] = tc_dense_nt(rows, N); row0[l] = l == 0 ? r0 : 0; bytes[l] = tc_plan_image_bytes((K + 63) & ~63, N); }
        }
        return PSA_OK;
    }
    PSA_REQUIRE(usage == PSA_USAGE_SA_MODULE, "mlp_image_plan: unknown usage %d", usage);
    TcArgs a;
    if (!tc_sa_eligible(mlp, c, nsample, &a)) return PSA_OK;
    if (c > 0 && dense_on_tc(rows, c, a.C1, 1)) { nt[0] = tc_dense_nt(rows, a.C1); row0[0] = 3; bytes[0] = tc_plan_image_bytes((c + 63) & ~63, a.C1); }
    for (int l = 0; l < a.nl; ++l) { nt[1 + l] = tc_sa_image_nt(); row0[1 + l] = 0; bytes[1 + l] = tc_plan_image_bytes(a.Kd[l], a.Ntot[l]); }
    return PSA_OK;
}
