// knn_tc.cu -- DGCNN's kNN graph (pairwise_distance + top_k, dgcnn/utils/tf_util.py:638-671) with the X.X^T contraction on
// the Hopper tensor cores (wgmma) and an EXACT refine, so the neighbour indices stay bit-identical to the canonical fp32 evaluation
// (oracle/psa_oracle.c orc_dgcnn_knn: dot as an fma chain over the channels, adj = (|p|^2 + (-2 dot)) + |q|^2, k smallest,
// lower index first on ties).
//
//   prep      a translation vector per cloud (knn_centre_kernel); every point row minus that vector is split once into bf16 pieces
//             and laid out as [128 rows][64 k] K-major SWIZZLE_128B blocks (the weight-image layout of tc_mlp.cu), + the
//             canonical |x|^2 and the centred |x - mu|^2 per row;
//   main      CTA = 128 query rows of one cloud.  The query block is the A operand, candidate blocks stream through a two-stage
//             ring (cp.async.bulk, one loader warp) as the B operand; four warpgroups each compute one 64 x 64 quarter of the
//             G tile with wgmma and consume it straight from their accumulator registers (two rows x 16 columns per thread):
//     pass 1  one bf16 MMA term (4 MMAs per tile): coarse distances (error <= E1) -> per-row histogram over logarithmic bins
//             (float exponent + 4 mantissa bits) in shared memory -> tau = upper edge of the bin that holds the k-th smallest;
//     pass 2  six MMA terms (bf16x3, error <= E2): every candidate with d < tau + E1 + E2 -- a superset of the true top-k -- is
//             appended to the row's list (typically k + 10..30 entries);
//     order   rank of every listed candidate = its output position.  Fine distances decide wherever two entries are more than
//             2 E2 apart; entries with a neighbour inside 2 E2 (near-ties, duplicates) get their canonical fp32 distance and are
//             compared canonically (distance, then index) -- every comparison agrees with the canonical order.
//   fallback  rows whose list overflows (many equidistant points) or whose cloud holds non-finite values are written to a
//             worklist and done exhaustively in fp32 by knn_rows_exact_kernel (same canonical arithmetic).
#include <float.h>

#include "common.cuh"
#include "tc_common.cuh"

// pass 2 precision: 6 = three bf16 pieces per operand (bf16x3, default), 3 = two pieces (a1 b1 + a1 b2 + a2 b1).
// The ordering step relies on |fine - canonical| <= E2 with E2 = 1e-4 |q||c| (+ the canonical formula's own rounding), so the bound has
// to be rigorous.  Per distance (= -2 x the Gram entry): six terms drop <= 2 * 4 * 2^-24 |q||c| of products and add <= 2 * 24 MMAs *
// 17 * 2^-23 |q||c| of truncating accumulation = 9.3e-5 in the worst case (measured: 0.005 E2).  Three terms drop 2 * 3 * 2^-16 = 9.2e-5
// of products ALONE (bf16 rounds to 2^-8) -- 1.4e-4 with the accumulation, above the bound (measured up to 0.33 E2 on 3-D clouds) -- and
// run only 5 % faster (352 vs 374 us at B=32 N=2048 C=64): a build with PSA_KNN_TERMS=3 must also raise E2 to 1.5e-4.
#ifndef PSA_KNN_TERMS
#define PSA_KNN_TERMS 6
#endif

namespace psa {
using namespace tc;

constexpr int kKtRowT = 4;                        // threads per query row (each owns 128 / kKtRowT columns of every tile)
constexpr int kKtThreads = 128 * kKtRowT + 32;    // row warps (four warpgroups) + 1 loader warp
constexpr uint32_t kKtPiece = 128u * 128u;        // one bf16 piece of a [128 rows][64 k] block: 16 KB
constexpr uint32_t kKtBlock = 3u * kKtPiece;      // 48 KB
constexpr int kKtBins = 256;
constexpr int kKtCap = 96;                        // list entries per row
constexpr int kKtMaxN = 2048;                     // candidates per cloud on this path (shared-memory budget)

// ---- centre: a translation vector per cloud (mean of every 8th point, fixed order).  Distances do not depend on it mathematically;
// the tensor-core passes run on x - mu so that their error bounds scale with the cloud's EXTENT, not with its offset from the origin
// (post-ReLU feature clouds sit far from it: |x|^2 ~ 100 x the neighbour distances, and bounds relative to |x|^2 would admit
// hundreds of candidates per row).  Any vector works -- the canonical refine always uses the original coordinates. ----
constexpr int kKtMeanLanes = 16;
__global__ void __launch_bounds__(64 * kKtMeanLanes) knn_centre_kernel(int n, int c, const float* __restrict__ x, float* __restrict__ mu) {
    __shared__ float s_part[kKtMeanLanes][64];
    const int cloud = blockIdx.x, ch = threadIdx.x & 63, rl = threadIdx.x >> 6;
    float s = 0.f;
    int cnt = 0;
    if (ch < c)
        for (int r = rl * 8; r < n; r += 8 * kKtMeanLanes) { s += __ldg(x + ((size_t)cloud * n + r) * c + ch); ++cnt; }
    s_part[rl][ch] = s;
    __shared__ int s_cnt[kKtMeanLanes];
    if (ch == 0) s_cnt[rl] = cnt;
    __syncthreads();
    if (rl == 0) {
        float t = 0.f;
        int m = 0;
        for (int i = 0; i < kKtMeanLanes; ++i) { t += s_part[i][ch]; m += s_cnt[i]; }
        mu[cloud * 64 + ch] = ch < c ? t / (float)max(m, 1) : 0.f;
    }
}

// ---- prep: block = 128 rows.  Phase A: thread = row, the canonical |x|^2 (sequential fma chain) and the centred |x - mu|^2.
// Phase B: warp = row, lane = two consecutive channels: coalesced 256-byte reads, three packed bf16x2 words of x - mu per lane into
// the swizzled rows ----
__global__ void __launch_bounds__(128) knn_prep_kernel(int n, int npad, int c, const float* __restrict__ x, const float* __restrict__ mu,
                                                       uint8_t* __restrict__ image, float* __restrict__ sq, float* __restrict__ sqc) {
    const int cloud = blockIdx.y, rb = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint8_t* blk = image + ((size_t)cloud * (npad / 128) + rb) * kKtBlock;
    __shared__ float s_mu[64];
    if (tid < 64) s_mu[tid] = mu[cloud * 64 + tid];
    __syncthreads();
    {
        const int r = rb * 128 + tid;
        float s = __int_as_float(0x7f800000), sc = __int_as_float(0x7f800000);
        if (r < n) {
            const float* xr = x + ((size_t)cloud * n + r) * c;
            s = 0.f; sc = 0.f;
            if ((c & 3) == 0 && (reinterpret_cast<uintptr_t>(xr) & 15) == 0) {
                for (int l = 0; l < c; l += 4) {
                    const float4 v = __ldg(reinterpret_cast<const float4*>(xr + l));
                    s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
                    const float d0 = v.x - s_mu[l], d1 = v.y - s_mu[l + 1], d2 = v.z - s_mu[l + 2], d3 = v.w - s_mu[l + 3];
                    sc = fmaf(d0, d0, sc); sc = fmaf(d1, d1, sc); sc = fmaf(d2, d2, sc); sc = fmaf(d3, d3, sc);
                }
            } else {
                for (int l = 0; l < c; ++l) { const float v = __ldg(xr + l); s = fmaf(v, v, s); const float d = v - s_mu[l]; sc = fmaf(d, d, sc); }
            }
        }
        sq[(size_t)cloud * npad + r] = s;
        sqc[(size_t)cloud * npad + r] = sc;
    }
    for (int rr = warp * 32; rr < warp * 32 + 32; ++rr) {
        const int r = rb * 128 + rr, k = 2 * lane;
        float h0 = 0.f, h1 = 0.f;
        if (r < n) {
            const float* xr = x + ((size_t)cloud * n + r) * c;
            if (k < c) h0 = __ldg(xr + k) - s_mu[k];
            if (k + 1 < c) h1 = __ldg(xr + k + 1) - s_mu[k + 1];
        }
        const uint32_t off = swz_off_bf16((uint32_t)rr, (uint32_t)k, 128u);
        const uint32_t p1 = pack_bf16x2(h0, h1);
        h0 -= __uint_as_float(p1 << 16); h1 -= __uint_as_float(p1 & 0xffff0000u);
        const uint32_t p2 = pack_bf16x2(h0, h1);
        h0 -= __uint_as_float(p2 << 16); h1 -= __uint_as_float(p2 & 0xffff0000u);
        const uint32_t p3 = pack_bf16x2(h0, h1);
        *reinterpret_cast<uint32_t*>(blk + off) = p1;
        *reinterpret_cast<uint32_t*>(blk + kKtPiece + off) = p2;
        *reinterpret_cast<uint32_t*>(blk + 2u * kKtPiece + off) = p3;
    }
}

struct KnnTcArgs {
    int n, npad, c, k;
    const float* x;
    const uint8_t* image;
    const float* sq;           // (b, npad) canonical |x|^2 (the refine and the exhaustive kernel)
    const float* sqc;          // (b, npad) |x - mu|^2 (the tensor-core passes)
    int* nn_idx;
    int* flag_rows;            // (b * n) worklist of global row ids for the exhaustive kernel
    unsigned* flag_count;
};

// canonical distance of the oracle: dot = fma chain over the channels, adj = (sq_p + (-2 dot)) + sq_q
__device__ __forceinline__ float knn_canonical(const float* __restrict__ xp, const float* __restrict__ xq, int c, float sqp, float sqq) {
    float dot = 0.f;
    if ((c & 3) == 0 && ((reinterpret_cast<uintptr_t>(xp) | reinterpret_cast<uintptr_t>(xq)) & 15) == 0) {
        for (int l = 0; l < c; l += 4) {                 // same ascending-channel fma chain, 16-byte loads
            const float4 u = __ldg(reinterpret_cast<const float4*>(xp + l)), v = __ldg(reinterpret_cast<const float4*>(xq + l));
            dot = fmaf(u.x, v.x, dot); dot = fmaf(u.y, v.y, dot); dot = fmaf(u.z, v.z, dot); dot = fmaf(u.w, v.w, dot);
        }
    } else {
        for (int l = 0; l < c; ++l) dot = fmaf(__ldg(xp + l), __ldg(xq + l), dot);
    }
    return __fadd_rn(__fadd_rn(sqp, __fmul_rn(-2.0f, dot)), sqq);
}

__global__ void __launch_bounds__(kKtThreads, 1) knn_tc_kernel(const __grid_constant__ KnnTcArgs a) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_qfull, s_full[2], s_dfree[2];
    __shared__ float s_wmax[kKtThreads / 32], s_wmaxo[kKtThreads / 32];
    __shared__ float s_T[128];
    __shared__ int s_cnt[128], s_namb[128];
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp_u = (int)warp_uniform((uint32_t)(tid >> 5));
    const int cloud = blockIdx.y;
    const int n = a.n, npad = a.npad, NT = npad / 128;
    uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* qblk = base;                                        // 48 KB
    uint8_t* cstage = base + kKtBlock;                           // 2 x 48 KB
    float* s_sq = reinterpret_cast<float*>(base + 3 * kKtBlock); // npad floats
    uint8_t* scratch = reinterpret_cast<uint8_t*>(s_sq + npad);  // pass 1: u16 hist[256][128]; pass 2: u16 idx[96][128] | float adj[96][128]
    unsigned* hist = reinterpret_cast<unsigned*>(scratch);      // [256 bins][64 words]: thread t counts in half (t >> 6) of word t & 63
    unsigned short* lidx = reinterpret_cast<unsigned short*>(scratch);
    float* ladj = reinterpret_cast<float*>(scratch + (size_t)kKtCap * 128 * 2);
    const uint8_t* img = a.image + (size_t)cloud * NT * kKtBlock;
    const float* sqc = a.sqc + (size_t)cloud * npad;      // centred norms: what the tensor-core distances are assembled from
    const float* sqo = a.sq + (size_t)cloud * npad;       // original norms: the canonical formula and its rounding bound

    if (tid == 0) {
        mbar_init(&s_qfull, 1);
        for (int i = 0; i < 2; ++i) { mbar_init(&s_full[i], 1); mbar_init(&s_dfree[i], 4 * kKtRowT); }
        fence_mbar_init();
    }
    // candidate norms -> shared memory; the cloud's largest finite-or-not norm over the real points
    float mx = 0.f, mxo = 0.f;
    for (int i = tid; i < npad; i += kKtThreads) {
        const float v = __ldg(sqc + i), vo = __ldg(sqo + i);
        s_sq[i] = v;
        if (i < n) {
            mx = fmaxf(mx, fabsf(v) <= FLT_MAX ? v : __int_as_float(0x7f800000));            // NaN -> +inf: the cloud is flagged
            mxo = fmaxf(mxo, fabsf(vo) <= FLT_MAX ? vo : __int_as_float(0x7f800000));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); mxo = fmaxf(mxo, __shfl_xor_sync(0xffffffffu, mxo, o)); }
    if (lane == 0) { s_wmax[warp_u] = mx; s_wmaxo[warp_u] = mxo; }
    __syncthreads();
    // pass 1 could look at a subset of the tiles (the k-th smallest of a SUBSET is still an upper bound of the k-th smallest of the
    // cloud): measured, every second tile halves the histogram work but doubles the lists -- 1-3 % of the rows of a feature cloud then
    // overflow kKtCap and the exhaustive kernel costs more than was saved (716 -> 1218 us at C = 64).  So: every tile.
    constexpr int kStride1 = 1;
    const int NT1 = (NT + kStride1 - 1) / kStride1;
    const int J = NT1 + NT;                          // jobs: pass 1 tiles (0, 2, 4, ..), then every pass 2 tile

    constexpr uint32_t kTermPieces = PSA_KNN_TERMS == 6 ? 3u : 2u;
    if (warp_u == 4 * kKtRowT) {
        // ================= loader warp =================
        auto load = [&](int j) {
            const int s = j & 1, t = j < NT1 ? kStride1 * j : j - NT1;
            const uint32_t bytes = j < NT1 ? kKtPiece : (kTermPieces * kKtPiece);   // pass 1 needs the leading piece only
            mbar_expect_tx(&s_full[s], bytes);
            for (uint32_t o = 0; o < bytes; o += 16384u) bulk_g2s(cstage + (uint32_t)s * kKtBlock + o, img + (size_t)t * kKtBlock + o, 16384u, &s_full[s]);
        };
        if (lane == 0) {
            mbar_expect_tx(&s_qfull, kKtBlock);
            for (uint32_t o = 0; o < kKtBlock; o += 16384u) bulk_g2s(qblk + o, img + (size_t)blockIdx.x * kKtBlock + o, 16384u, &s_qfull);
            load(0);
            if (J > 1) load(1);
            for (int j = 0; j + 2 < J; ++j) {
                mbar_wait(&s_dfree[j & 1], (uint32_t)((j >> 1) & 1));     // every warpgroup's MMAs of job j are done: refill two jobs ahead
                load(j + 2);
            }
        }
    } else {
        // ================= row threads: kKtRowT threads per query row =================
        // In the two passes every thread consumes its own wgmma fragment (two rows x 16 columns of a 64 x 64 quarter of the tile); in the
        // per-row work after them, thread (r, h) = (tid & 127, tid >> 7) is one of the kKtRowT threads of query row r.  Histogram counters
        // and the candidate list of a row are shared by all threads that touch the row through shared-memory atomics.
        const int r = tid & 127, h = tid >> 7;
        const int q = blockIdx.x * 128 + r;
        const bool valid = q < n;
        float sqmax = s_wmax[0], sqmaxo = s_wmaxo[0];
#pragma unroll
        for (int w = 1; w < kKtThreads / 32; ++w) { sqmax = fmaxf(sqmax, s_wmax[w]); sqmaxo = fmaxf(sqmaxo, s_wmaxo[w]); }
        const float sqq = s_sq[valid ? q : 0];                 // centred
        const float sqqo = __ldg(sqo + (valid ? q : 0));       // original
        const bool ok = valid && fabsf(sqq) <= FLT_MAX && fabsf(sqmax) <= FLT_MAX && fabsf(sqqo) <= FLT_MAX && fabsf(sqmaxo) <= FLT_MAX;
        const float sgeo = sqrtf(sqq * sqmax);
        // |fine - canonical| <= E2: the bf16 products and fp32 sums of the centred Gram entry (relative to the centred norms) + what the
        // canonical fp32 formula itself loses on the ORIGINAL coordinates (its 64-term dot chain and two adds; centring rounds too)
        const float E2 = (PSA_KNN_TERMS == 6 ? 1e-4f : 1.5e-4f) * sgeo + 8e-6f * sqrtf(sqqo * sqmaxo) + 2e-6f * (sqqo + sqmaxo);
        const float dmax = 2.0f * (sqq + sqmax);
        const int keymax = (int)(__float_as_uint(fmaxf(dmax, 1e-30f)) >> 19) + 1;
        constexpr int kRowThreads = 128 * kKtRowT;
        static_assert(kKtRowT == 4, "four warpgroups, one 64 x 64 quarter of every tile each");
        // G tile of job j: warpgroup h computes rows 64 (h & 1) .., columns 64 (h >> 1) ..; this thread holds rows fr[0], fr[1] and
        // columns 64 (h >> 1) + 8 i + 2 t + e of d[4 i + 2 u + e] (u = row), see tc_common.cuh
        const int g = lane >> 2, tq = lane & 3;
        const int fr[2] = {(h & 1) * 64 + (warp_u & 3) * 16 + g, (h & 1) * 64 + (warp_u & 3) * 16 + g + 8};
        const int fc0 = (h >> 1) * 64 + 2 * tq;
        float fsq[2];
        int fkeymax[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int fq = blockIdx.x * 128 + fr[u];
            fsq[u] = s_sq[fq < n ? fq : 0];
            fkeymax[u] = (int)(__float_as_uint(fmaxf(2.0f * (fsq[u] + sqmax), 1e-30f)) >> 19) + 1;
        }
#if PSA_KNN_TERMS == 6
        constexpr uint32_t qp[6] = {0, 1, 2, 0, 1, 0};       // query piece / candidate piece of the terms, small products first
        constexpr uint32_t cp[6] = {2, 1, 0, 1, 0, 0};
#else
        constexpr uint32_t qp[3] = {0, 1, 0};
        constexpr uint32_t cp[3] = {1, 0, 0};
#endif
        // all four k-steps of the 64-channel block, whatever c is: the image is zero beyond c, so the extra products are exact zeros,
        // and a fixed count keeps the wgmma sequence straight-line (a runtime trip count makes ptxas serialise it)
        constexpr int ks = 4;
        const uint32_t qa = smem_u32(qblk) + (uint32_t)(h & 1) * 8192u;
        // the MMAs of job j into d (waits for the stage; tells the loader when the stage may be refilled)
        auto gram = [&](int j, bool fine, float (&d)[32]) {
            const int s = j & 1;
            mbar_wait(&s_full[s], (uint32_t)((j >> 1) & 1));
            const uint32_t cb = smem_u32(cstage) + (uint32_t)s * kKtBlock + (uint32_t)(h >> 1) * 8192u;
            wg_fence();
            if (!fine) {
#pragma unroll
                for (int s4 = 0; s4 < ks; ++s4) wg_mma_ss_bf16(d, wg_desc(qa + s4 * 32), wg_desc(cb + s4 * 32), s4 ? 1u : 0u);
            } else {
#pragma unroll
                for (int t6 = 0; t6 < PSA_KNN_TERMS; ++t6)
#pragma unroll
                    for (int s4 = 0; s4 < ks; ++s4)
                        wg_mma_ss_bf16(d, wg_desc(qa + qp[t6] * kKtPiece + s4 * 32), wg_desc(cb + cp[t6] * kKtPiece + s4 * 32), (t6 | s4) ? 1u : 0u);
            }
            wg_commit();
            wg_wait_all();
            wg_fence_acc(d);
            __syncwarp();
            if (lane == 0) mbar_arrive1(&s_dfree[s]);
        };
        for (int b = tid; b < kKtBins * 64; b += kRowThreads) hist[b] = 0u;
        if (h == 0) { s_cnt[r] = 0; s_namb[r] = 0; }
        mbar_wait(&s_qfull, 0);
        asm volatile("bar.sync 2, %0;" ::"n"(128 * kKtRowT) : "memory");
        // ---- pass 1: coarse distances -> histogram ----
        // (A running cut -- skipping the atomics of candidates farther than the bins that already hold k -- costs more in predicated
        //  atomics and periodic histogram scans than the atomics it saves.)
        for (int t1 = 0; t1 < NT1; ++t1) {
            const int t = kStride1 * t1;
            float d[32];
            gram(t1, false, d);
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int u = 0; u < 2; ++u)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float dist = fmaf(-2.0f, d[4 * i + 2 * u + e], fsq[u] + s_sq[t * 128 + fc0 + 8 * i + e]);
                        const int key = __float_as_int(dist) >> 19;      // arithmetic shift: zero / negative distances land in the last (nearest) bin
                        const int bin = min(max(fkeymax[u] - key, 0), kKtBins - 1);
                        atomicAdd(hist + (fr[u] & 63) + bin * 64, fr[u] < 64 ? 1u : 65536u);     // fire-and-forget
                    }
        }
        asm volatile("bar.sync 2, %0;" ::"n"(128 * kKtRowT) : "memory");           // every row's histogram is complete
        // ---- threshold: upper edge of the bin that holds the k-th smallest coarse distance, widened by the error bounds ----
        if (h == 0) {
            const unsigned* hcol = hist + (r & 63);
            int cum = 0, b = kKtBins - 1;
            for (; b >= 0; --b) { const unsigned w = hcol[b * 64]; cum += (int)(r < 64 ? (w & 0xffffu) : (w >> 16)); if (cum >= a.k) break; }
            const float tau = b < 0 ? __int_as_float(0x7f800000) : __uint_as_float((uint32_t)(keymax - b + 1) << 19);
            // |coarse - exact| <= E1 (one bf16 term: 2^-8 relative on every product), |fine - exact| <= E2 (bf16x3 + fp32 sums)
            const float E1 = 0.01f * sgeo;
            s_T[r] = tau + E1 + E2 + 1e-6f * tau;
        }
        // every row is done with its histogram before anybody's candidate list / distances overwrite the scratch area
        asm volatile("bar.sync 2, %0;" ::"n"(128 * kKtRowT) : "memory");
        const float fT[2] = {s_T[fr[0]], s_T[fr[1]]};
        // ---- pass 2: fine distances -> the row's candidate list (slots handed out by a shared-memory counter) ----
        for (int t = 0; t < NT; ++t) {
            float d[32];
            gram(NT1 + t, true, d);
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int u = 0; u < 2; ++u)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = fc0 + 8 * i + e;
                        const float dist = fmaf(-2.0f, d[4 * i + 2 * u + e], fsq[u] + s_sq[t * 128 + col]);
                        if (dist < fT[u]) {
                            const int slot = atomicAdd(&s_cnt[fr[u]], 1);
                            if (slot < kKtCap) {
                                lidx[slot * 128 + fr[u]] = (unsigned short)(t * 128 + col);
                                ladj[slot * 128 + fr[u]] = dist;
                            }
                        }
                    }
        }
        asm volatile("bar.sync 2, %0;" ::"n"(128 * kKtRowT) : "memory");
        const int cnt = s_cnt[r];
        const bool refine = ok && cnt <= kKtCap && cnt >= a.k;
        if (valid && !refine && h == 0) {
            // exhaustive kernel takes this row (overflow: many equidistant candidates; non-finite coordinates; fewer than k below T)
            a.flag_rows[atomicAdd(a.flag_count, 1u)] = cloud * n + q;
        }
        // ---- order of the listed candidates.  The fine distances are within E2 of the canonical fp32 values, so two entries more
        // than delta = 2 E2 apart are ordered canonically the way their fine distances are; only entries with a neighbour inside
        // delta ("ambiguous": near-ties, duplicates) get their canonical distance evaluated, and only those pairs are compared
        // canonically (distance, then index).  Every pairwise comparison therefore agrees with the canonical order and
        // rank = number of entries that precede = output position.  Typical feature clouds: 1-3 ambiguous entries per row instead of
        // 30-40 canonical evaluations (each a 256-byte gather).  The operand buffers are dead after pass 2 and hold the scratch:
        float* lcan = reinterpret_cast<float*>(qblk);                       // [kKtCap][128] canonical distance of ambiguous entries
        unsigned short* lrank = reinterpret_cast<unsigned short*>(cstage);   // [kKtCap][128] number of entries surely before
        unsigned char* lamb = cstage + (size_t)kKtCap * 128 * 2;             // [kKtCap][128] compact list of the row's ambiguous entries
        const float* xc = a.x + (size_t)cloud * n * a.c;
        const float delta = 2.0f * E2;
        int* out = a.nn_idx + ((size_t)cloud * n + q) * a.k;
        // phase 1: fine-distance counts of every entry (entries split between the row's threads); unambiguous ones are final
        if (refine) {
            for (int e = h; e < cnt; e += kKtRowT) {
                const float fe = ladj[e * 128 + r];
                int lo = 0, amb = 0;
#pragma unroll 4
                for (int f = 0; f < cnt; ++f) {
                    const float d = ladj[f * 128 + r] - fe;
                    lo += d < -delta ? 1 : 0;
                    amb += fabsf(d) <= delta ? 1 : 0;                        // counts e itself
                }
                if (amb == 1) {
                    if (lo < a.k) out[lo] = lidx[e * 128 + r];
                } else {
                    lrank[e * 128 + r] = (unsigned short)lo;
                    lamb[atomicAdd(&s_namb[r], 1) * 128 + r] = (unsigned char)e;
                }
            }
        }
        asm volatile("bar.sync 2, %0;" ::"n"(128 * kKtRowT) : "memory");
        // phase 2: canonical distances of the ambiguous entries, dealt round-robin to the row's threads
        const int namb = refine ? s_namb[r] : 0;
        if (namb > 0) {
            const float* xq = xc + (size_t)q * a.c;
            const bool wide = a.c == 64 && (reinterpret_cast<uintptr_t>(xc) & 15) == 0;
            for (int i = h; i < namb; i += kKtRowT) {
                const int e = lamb[i * 128 + r];
                const int col = lidx[e * 128 + r];
                float can;
                if (wide) {
                    // the usual DGCNN width: 2 x 8 independent 16-byte loads per operand, one ascending fma chain
                    const float4* cp4 = reinterpret_cast<const float4*>(xc + (size_t)col * 64);
                    const float4* qp4 = reinterpret_cast<const float4*>(xq);
                    float dot = 0.f;
#pragma unroll
                    for (int hf = 0; hf < 2; ++hf) {
                        float4 qv[8], cv[8];
#pragma unroll
                        for (int l = 0; l < 8; ++l) { qv[l] = __ldg(qp4 + hf * 8 + l); cv[l] = __ldg(cp4 + hf * 8 + l); }
#pragma unroll
                        for (int l = 0; l < 8; ++l) {
                            dot = fmaf(qv[l].x, cv[l].x, dot); dot = fmaf(qv[l].y, cv[l].y, dot);
                            dot = fmaf(qv[l].z, cv[l].z, dot); dot = fmaf(qv[l].w, cv[l].w, dot);
                        }
                    }
                    can = __fadd_rn(__fadd_rn(sqqo, __fmul_rn(-2.0f, dot)), __ldg(sqo + col));
                } else {
                    can = knn_canonical(xq, xc + (size_t)col * a.c, a.c, sqqo, __ldg(sqo + col));
                }
                lcan[e * 128 + r] = can;
            }
        }
        asm volatile("bar.sync 2, %0;" ::"n"(128 * kKtRowT) : "memory");
        // phase 3: an ambiguous entry is preceded by the entries surely before it plus the ambiguous neighbours that precede canonically
        for (int i = h; i < namb; i += kKtRowT) {
            const int e = lamb[i * 128 + r];
            const float fe = ladj[e * 128 + r], ce = lcan[e * 128 + r];
            const int ie = lidx[e * 128 + r];
            int rank = lrank[e * 128 + r];
            for (int j = 0; j < namb; ++j) {
                const int f = lamb[j * 128 + r];
                if (f == e || fabsf(ladj[f * 128 + r] - fe) > delta) continue;
                const float cf = lcan[f * 128 + r];
                const int jf = lidx[f * 128 + r];
                rank += (cf < ce || (cf == ce && jf < ie)) ? 1 : 0;
            }
            if (rank < a.k) out[rank] = ie;
        }
    }
}

// ---- exhaustive rows (worklist): one warp per row, canonical distances of all n candidates in shared memory, then k rounds of
// lexicographic minimum.  NaN distances are never selected ahead of numbers (the oracle's `row[q] < row[best]` is false for them).
constexpr int kKxWarps = 4;
__global__ void __launch_bounds__(kKxWarps * 32) knn_rows_exact_kernel(int n, int c, int k, const float* __restrict__ x, const float* __restrict__ sq,
                                                                      int npad, const int* __restrict__ rows, const unsigned* __restrict__ count,
                                                                      int* __restrict__ nn_idx) {
    extern __shared__ float sm_d[];                  // kKxWarps x n
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* dist = sm_d + (size_t)warp * n;
    const unsigned total = *count;
    for (unsigned w = blockIdx.x * kKxWarps + warp; w < total; w += gridDim.x * kKxWarps) {
        const int row = rows[w];
        const int cloud = row / n, p = row - cloud * n;
        const float* xc = x + (size_t)cloud * n * c;
        const float* sqc = sq + (size_t)cloud * npad;
        const float sqp = __ldg(sqc + p);
        for (int qd = lane; qd < n; qd += 32) dist[qd] = knn_canonical(xc + (size_t)p * c, xc + (size_t)qd * c, c, sqp, __ldg(sqc + qd));
        __syncwarp();
        int* out = nn_idx + (size_t)row * k;
        // the oracle scans q ascending keeping the first strict minimum among the untaken: equal values -> lowest index; a NaN
        // candidate is only ever chosen when it is the first untaken entry and nothing compares below it
        unsigned long long taken_lo = 0ull;          // (the general "taken" set lives in the NaN-free ordering below)
        (void)taken_lo;
        float pd = -__int_as_float(0x7f800000);
        int pi = -1;
        for (int r = 0; r < k; ++r) {
            float bd = __int_as_float(0x7f800000);
            int bi = 0x7fffffff;
            for (int qd = lane; qd < n; qd += 32) {
                const float dd = dist[qd];
                const bool after = dd > pd || (dd == pd && qd > pi);
                const bool better = dd < bd || (dd == bd && qd < bi);
                if (after && better) { bd = dd; bi = qd; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float od = __shfl_xor_sync(0xffffffffu, bd, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
            }
            if (bi == 0x7fffffff) {
                // only +inf / NaN entries remain beyond (pd, pi): take the lowest untaken index (the oracle's scan order)
                int cand = 0x7fffffff;
                for (int qd = lane; qd < n; qd += 32) {
                    const float dd = dist[qd];
                    const bool fin_after = dd > pd || (dd == pd && qd > pi);
                    bool used = false;
                    for (int u = 0; u < r; ++u) used = used || (out[u] == qd);
                    if (!used && !(fin_after && dd < __int_as_float(0x7f800000))) cand = min(cand, qd);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, o));
                bi = cand;
                bd = __int_as_float(0x7f800000);
            }
            if (lane == 0) out[r] = bi;
            __syncwarp();
            pd = bd; pi = bi;
        }
        __syncwarp();
    }
}

static size_t knn_tc_smem_bytes(int npad) {
    return 1024 + 3 * (size_t)kKtBlock + (size_t)npad * 4 + (size_t)kKtCap * 128 * 2 + (size_t)kKtCap * 128 * 4 + 64;
}

bool knn_tc_eligible(int n, int c, int k) { return n >= 128 && n <= kKtMaxN && c >= 1 && c <= 64 && k >= 1 && k <= 32; }   // tile 0 (128 real points) is in the pass-1 subsample: it holds k candidates

}  // namespace psa

using namespace psa;

extern "C" size_t psa_knn_graph_workspace_bytes(int b, int n, int c, int k) {
    if (!knn_tc_eligible(n, c, k)) return 0;
    const int npad = (n + 127) / 128 * 128;
    return (size_t)b * (npad / 128) * kKtBlock + 2 * (((size_t)b * npad * 4 + 255) & ~(size_t)255) + (((size_t)b * n * 4 + 255) & ~(size_t)255) + 256 +
           (((size_t)b * 64 * 4 + 255) & ~(size_t)255);
}

// fp32 kernel of graph.cu (no workspace)
extern "C" int psa_knn_graph(int b, int n, int c, int k, const float* x, int* nn_idx, psa_stream_t stream);

extern "C" int psa_knn_graph_ws(int b, int n, int c, int k, const float* x, int* nn_idx, void* workspace, size_t workspace_bytes,
                                psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 0 && c >= 0 && k >= 0, "knn_graph: negative dimension");
    PSA_REQUIRE(k <= n || b == 0, "knn_graph: k=%d exceeds the number of points n=%d", k, n);
    if (b == 0 || n == 0 || k == 0) return PSA_OK;
    const size_t need = psa_knn_graph_workspace_bytes(b, n, c, k);
    if (need == 0 || workspace == nullptr || workspace_bytes < need || b > 65535) return psa_knn_graph(b, n, c, k, x, nn_idx, stream);
    PSA_REQUIRE(x && nn_idx, "knn_graph: null buffer");
    cudaStream_t st = as_stream(stream);
    const int npad = (n + 127) / 128 * 128, NT = npad / 128;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    uint8_t* image = ws;
    ws += (size_t)b * NT * kKtBlock;
    float* sq = reinterpret_cast<float*>(ws);
    ws += ((size_t)b * npad * 4 + 255) & ~(size_t)255;
    int* flag_rows = reinterpret_cast<int*>(ws);
    ws += ((size_t)b * n * 4 + 255) & ~(size_t)255;
    unsigned* flag_count = reinterpret_cast<unsigned*>(ws);
    ws += 256;
    float* sqc = reinterpret_cast<float*>(ws);
    ws += ((size_t)b * npad * 4 + 255) & ~(size_t)255;
    float* mu = reinterpret_cast<float*>(ws);
    PSA_CUDA(cudaMemsetAsync(flag_count, 0, 4 * sizeof(unsigned), st));       // [0] worklist length
    knn_centre_kernel<<<b, 64 * kKtMeanLanes, 0, st>>>(n, c, x, mu);
    knn_prep_kernel<<<dim3(NT, b), 128, 0, st>>>(n, npad, c, x, mu, image, sq, sqc);
    int rc = check_launch("knn_prep_kernel");
    if (rc != PSA_OK) return rc;
    KnnTcArgs a;
    a.n = n; a.npad = npad; a.c = c; a.k = k; a.x = x; a.image = image; a.sq = sq; a.sqc = sqc; a.nn_idx = nn_idx; a.flag_rows = flag_rows; a.flag_count = flag_count;
    const size_t smem = knn_tc_smem_bytes(npad);
    PSA_CUDA(cudaFuncSetAttribute(knn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    knn_tc_kernel<<<dim3(NT, b), kKtThreads, smem, st>>>(a);
    rc = check_launch("knn_tc_kernel");
    if (rc != PSA_OK) return rc;
    const size_t xsmem = (size_t)kKxWarps * n * sizeof(float);
    PSA_CUDA(cudaFuncSetAttribute(knn_rows_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)xsmem));
    knn_rows_exact_kernel<<<2 * kNumSMs, kKxWarps * 32, xsmem, st>>>(n, c, k, x, sq, npad, flag_rows, flag_count, nn_idx);
    return check_launch("knn_rows_exact_kernel");
}
