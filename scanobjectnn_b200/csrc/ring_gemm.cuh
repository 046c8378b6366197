// ring_gemm.cuh -- the warp-specialised tensor-core GEMM shared by the dense layers (tc_mlp.cu), spiderConv (spider.cu), conv3d
// (mfv.cu) and PointCNN's dense layers (pointcnn.cu), its fp32-FMA fallback, and the host sequence that runs it under the fp16x2
// range guard.
//
// ring_gemm<NP, NC>(op, ring): per work unit, a 128-row x 64 NC-column tile of A . W, with A staged by the op.  Persistent: producers
// and consumers both walk units blockIdx.x, blockIdx.x + gridDim.x, ..., and a unit may have no K blocks.  An op with kClaim walks
// the same order when its launch carries no counter (RingArgs::counter); with one, units are claimed from it, so that a CTA that
// starts late or shares its SM with another stream's kernels simply takes fewer.  One producer lane claims each unit and shares it
// with the other producer warps, the unit's stages carry it to the consumers and a stage tagged -1 follows the last one; every
// claimed unit must have a K block.
// CTA = two consumer warpgroups (rows 0-63 / 64-127) + a producer warpgroup whose four warps each stage 32 rows of every 64-wide K
// block by cp.async while warp 0 also drops the block's weights in by TMA.  Consumers: per block one wgmma group on the registers
// prepared under the previous one, the block's sum added to fp32 accumulators (no tensor-core accumulation over more than 64 K).
// The ring holds as many stages as the op's shared-memory budget (kBudget) takes, at most 4.  168 registers per thread at launch:
// the 128 x 128 the producers release (setmaxnreg 40) are exactly the 256 x 64 the consumers take (232).  Named barrier 1 is the
// op's (the 256 consumer threads), 2 the claiming producers'.
//
// The op supplies what differs (Op::Smem is its shared table, Unit its per-unit consumer state):
//   kClaim, kBudget                                           units claimed from a counter; bytes of dynamic shared memory
//   int units(int Nt)                                         work units for Nt-wide column tiles
//   produce(unit, Nt, pw, lane, Smem&, put)                   producer warp pw's share of a unit: for each K block in order,
//                                                             put(image block, stage) with stage(xs) issuing the cp.async copies
//                                                             of the warp's 32 rows into the staged block at shared address xs
//   Unit unit(unit, Nt, row, Smem&, n)                        .nb K blocks, .col0 first column; the thread's rows are row, row + 8;
//                                                             n: the unit's ordinal in the CTA
//   load(u, xs, kb, t, x)                                     staged block kb -> the A operand's values x[s][h][i] of the thread:
//                                                             row + 8 i, block columns 16 s + 8 h + 2 t, + 1 (staged_pair)
//   epilogue(u, acc, col, t, colscale, Smem&)                 a 64-column chunk of sums from column col (colscale: fp16x2 only)
// and for the FMA fallback, fma_gemm(op, ...): float load_a(row, k) and store(row, col, sum).
#pragma once
#include "common.cuh"
#include "mlp_internal.cuh"
#include "tc_common.cuh"

namespace psa {

// the fields every ring launch carries: the weight image and the fp16x2 range guard (Split<NP>, tc_common.cuh)
struct RingArgs {
    const uint8_t* image = nullptr;         // W in the format of NP, tile width 64 NC
    unsigned int* ovf = nullptr;            // np = 2: raised when an operand left the fp16 range or a weight is not finite
    const unsigned int* run_if = nullptr;   // non-null: no-op unless *run_if != 0
    const unsigned int* wflag = nullptr;    // np = 2: the image's non-finite-weight word
    const float* colscale = nullptr;        // np = 2: the image's column factors
    unsigned int* counter = nullptr;        // kClaim ops: zeroed before the launch, units are claimed from it; null: the fixed walk
};

constexpr int kRingThreads = 384, kRingConsumers = 256;
constexpr uint32_t kRingXRow = 64u * 4u + 32u;            // bytes per staged x row: 8-bank offset between rows g and g + 1
constexpr uint32_t kRingXBytes = 128u * kRingXRow;
constexpr uint32_t kRingBudget = 206u * 1024u;            // the spiderConv, conv3d and PointCNN ops' budget
__host__ __device__ constexpr uint32_t ring_stage_bytes(int NP, int NC) { return tc::tc_block_bytes(64 * NC, NP) + kRingXBytes; }
__host__ __device__ constexpr int ring_stages(int NP, int NC, uint32_t budget) {
    return budget / ring_stage_bytes(NP, NC) < 4u ? (int)(budget / ring_stage_bytes(NP, NC)) : 4;
}
static_assert(ring_stages(2, 1, kRingBudget) == 3 && ring_stages(3, 1, kRingBudget) == 3 && ring_stages(2, 2, kRingBudget) == 3 &&
              ring_stages(3, 2, kRingBudget) == 2, "stages of the spiderConv, conv3d and PointCNN rings");

// the 16-byte copies of a warp's rows [r0, r0 + nr) of K block kb of x (row stride ldx, K % 4 == 0) into the staged block at xs:
// lane (row half, 16-byte chunk), chunks past K not copied
__device__ __forceinline__ void stage_rows16(uint32_t xs, const float* x, long long ldx, long long row0, int r0, int nr, int kb, int K, int lane) {
    const int cc = (lane & 15) * 4, kk = kb * 64 + cc;
    if (kk >= K) return;
    for (int r = lane >> 4; r < nr; r += 2) {
        const int row = r0 + r;
        tc::cp_async16(xs + (uint32_t)row * kRingXRow + (uint32_t)cc * 4u, x + (size_t)(row0 + row) * ldx + kk);
    }
}

// the staged pair of row + 8 i, block columns 16 s + 8 h + 2 t, + 1; xs = the staged block's row `row`
__device__ __forceinline__ float2 staged_pair(const float* xs, int s, int h, int i, int t) {
    return *reinterpret_cast<const float2*>(xs + 8 * i * (int)(kRingXRow / 4) + 16 * s + 8 * h + 2 * t);
}

template <int NP, int NC, class Op>
__device__ __forceinline__ void ring_gemm(const Op& op, const RingArgs& ra) {
    using namespace tc;
    if (ra.run_if != nullptr && *ra.run_if == 0u) return;
    constexpr int Nt = 64 * NC, S = ring_stages(NP, NC, Op::kBudget);
    constexpr uint32_t bb = tc_block_bytes(Nt, NP), piece = Nt * 128u, SB = ring_stage_bytes(NP, NC);
    static_assert(S >= 2, "the ring needs two stages");
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_full[S], s_empty[S];
    __shared__ int s_tag[S], s_claim[2];                            // kClaim: the unit of a stage (-1: no more), a claimed unit
    __shared__ typename Op::Smem s_op;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int units = op.units(Nt);
    if (tid == 0) {
        for (int i = 0; i < S; ++i) { mbar_init(&s_full[i], 1 + 128); mbar_init(&s_empty[i], kRingConsumers / 32); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp >= kRingConsumers / 32) {
        // ---- producers: warp pw stages tile rows [32 pw, 32 pw + 32) ----
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
        const int pw = warp - kRingConsumers / 32;
        uint32_t q = 0;                                             // ring uses
        int cur = 0;                                                // kClaim: the unit being staged
        auto put = [&](size_t block, auto&& stage) {
            const int s = (int)(q % S);
            if (q >= (uint32_t)S) mbar_wait(&s_empty[s], ((q / S) - 1u) & 1u);
            if (pw == 0 && lane == 0) {
                if constexpr (Op::kClaim) s_tag[s] = cur;
                mbar_expect_tx(&s_full[s], bb);
                const uint8_t* src = ra.image + block * bb;
                for (uint32_t o = 0; o < bb; o += 16384u) bulk_g2s(base + (uint32_t)s * SB + o, src + o, min(16384u, bb - o), &s_full[s]);
            }
            stage(smem_u32(base + (uint32_t)s * SB + bb));
            cp_async_mbar_arrive(&s_full[s]);
            ++q;
        };
        if constexpr (Op::kClaim) {
            for (uint32_t n = 0;; ++n) {
                // by parity: a slower warp may still read the previous claim, but not the one before it
                if (pw == 0 && lane == 0) s_claim[n & 1] = ra.counter != nullptr ? (int)atomicAdd(ra.counter, 1u) : (int)(blockIdx.x + n * gridDim.x);
                unit_bar_sync(2, kRingThreads - kRingConsumers);
                cur = s_claim[n & 1];
                if (cur >= units) break;
                op.produce(cur, Nt, pw, lane, s_op, put);
            }
            const int s = (int)(q % S);                             // the end tag, a stage without data
            if (q >= (uint32_t)S) mbar_wait(&s_empty[s], ((q / S) - 1u) & 1u);
            if (pw == 0 && lane == 0) { s_tag[s] = -1; mbar_arrive1(&s_full[s]); }
            cp_async_mbar_arrive(&s_full[s]);
        } else {
            for (int unit = blockIdx.x; unit < units; unit += gridDim.x) op.produce(unit, Nt, pw, lane, s_op, put);
        }
        return;
    }

    // ---- consumers: warp w holds tile rows 16w + g and 16w + g + 8 ----
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
    const int g = lane >> 2, t = lane & 3, row = warp * 16 + g;
    uint32_t ovf = 0u;
    uint32_t q = 0;                                                 // ring uses
    for (int unit = blockIdx.x, n = 0;; unit += gridDim.x, ++n) {
        if constexpr (Op::kClaim) {
            mbar_wait(&s_full[q % S], (q / S) & 1u);
            unit = s_tag[q % S];
            if (unit < 0) break;
        } else if (unit >= units) {
            break;
        }
        const auto u = op.unit(unit, Nt, row, s_op, n);

        // staged block of ring use `use` -> the op's values -> A fragments
        auto prep = [&](uint32_t (&A)[NP][4][4], uint32_t use, int kb) {
            const float* xs = reinterpret_cast<const float*>(base + (use % S) * SB + bb) + row * (int)(kRingXRow / 4);
            float2 x[4][2][2];
            op.load(u, xs, kb, t, x);
#pragma unroll
            for (int s = 0; s < 4; ++s)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        uint32_t pc[NP];
                        split_pair<NP>(x[s][h][i].x, x[s][h][i].y, pc, ovf);
#pragma unroll
                        for (int e = 0; e < NP; ++e) A[e][s][i + 2 * h] = pc[e];
                    }
        };
        float acc[NC][32];
        // block kb (ring use `use`): issue its group on A, prepare block kb + 1 into An while it runs, wait, release the stage, add.
        // One group in flight, so every wait retires the same group on every path.  bf16x3 128-wide tiles issue one 64-channel chunk
        // per group (the next block is prepared under the second), so that two A buffers, the accumulators and one chunk's sum fit
        // the consumers' 232 registers.
        constexpr int CG = NP == 3 && NC == 2 ? 1 : NC;            // 64-channel chunks per group
        auto step = [&](const uint32_t (&A)[NP][4][4], uint32_t (&An)[NP][4][4], uint32_t use, int kb) {
            const uint32_t wb = smem_u32(base + (use % S) * SB);
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
                if (c0 + CG == NC && kb + 1 < u.nb) {
                    mbar_wait(&s_full[(use + 1) % S], ((use + 1) / S) & 1u);
                    prep(An, use + 1, kb + 1);
                }
                wg_wait_all();
                if (c0 + CG == NC) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive1(&s_empty[use % S]);
                }
#pragma unroll
                for (int c = 0; c < CG; ++c) {
                    wg_fence_acc(d[c]);
#pragma unroll
                    for (int e = 0; e < 32; ++e) acc[c0 + c][e] = kb ? acc[c0 + c][e] + d[c][e] : d[c][e];
                }
            }
        };
        if (u.nb > 0) {
            uint32_t A0[NP][4][4], A1[NP][4][4];
            mbar_wait(&s_full[q % S], (q / S) & 1u);
            prep(A0, q, 0);
            for (int kb = 0;; kb += 2) {
                step(A0, A1, q + kb, kb);
                if (kb + 1 == u.nb) break;
                step(A1, A0, q + kb + 1, kb + 1);
                if (kb + 2 == u.nb) break;
            }
            q += u.nb;
        } else {
#pragma unroll
            for (int c = 0; c < NC; ++c)
#pragma unroll
                for (int e = 0; e < 32; ++e) acc[c][e] = 0.f;
        }
        // one 64-column chunk at a time, its accumulators passed by reference (a loop over chunks indexes acc through the stack)
        const float* cs = NP == 2 ? ra.colscale : nullptr;
        op.epilogue(u, acc[0], u.col0, t, cs, s_op);
        if constexpr (NC == 2) op.epilogue(u, acc[1], u.col0 + 64, t, cs, s_op);
    }
    if constexpr (NP == 2) {
        if (f16x2_overflowed(ovf) || (tid == 0 && ra.wflag != nullptr && *ra.wflag != 0u)) atomicOr(ra.ovf, 1u);
    }
}

// C (rows, N) = A (rows, K) . W (K, N) on the fp32 FMA pipe: 64 x 64 tiles, 256 threads of 4 x 4 outputs, K in steps of 16, each
// 64-wide K block summed on its own before it is added to the total (as the ring sums).  op.load_a(row, k) is called inside the
// matrix only; op.store(row, col, sum) writes an output.
template <class Op>
__device__ __forceinline__ void fma_gemm(const Op& op, long long rows, int K, int N, const float* __restrict__ W) {
    __shared__ float As[16][64 + 4], Bs[16][64];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const long long row0 = (long long)blockIdx.x * 64;
    const int col0 = blockIdx.y * 64;
    float tot[4][4] = {}, part[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int e = tid + 256 * i, kr = e >> 6, rr = e & 63;
            const int kk = k0 + kr;
            const long long p = row0 + rr;
            As[kr][rr] = (kk < K && p < rows) ? op.load_a(p, kk) : 0.f;
            const int col = col0 + rr;
            Bs[kr][rr] = (kk < K && col < N) ? __ldg(W + (size_t)kk * N + col) : 0.f;
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
        if ((k0 & 63) == 48 || k0 + 16 >= K) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) { tot[i][jj] += part[i][jj]; part[i][jj] = 0.f; }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long p = row0 + ty * 4 + i;
        if (p >= rows) continue;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int col = col0 + tx * 4 + jj;
            if (col < N) op.store(p, col, tot[i][jj]);
        }
    }
}

// ---- host side ----
static inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

// an op's four ring kernels, fn[NP - 2][NC - 1], and the op's kBudget
struct RingKernels {
    const void* fn[2][2];
    const char* name;
    uint32_t budget;
};
// one launch of the (np, Nt / 64) kernel on min(units, SMs) CTAs; args points at the kernel's argument struct (ring_gemm.cu)
int ring_launch(const RingKernels& k, int np, int Nt, const void* args, long long units, cudaStream_t st);
// W (K, N) -> Wp (K, Np), columns N .. Np zero (mfv.cu)
int pad_cols(long long K, int N, int Np, const float* W, float* Wp, cudaStream_t st);

// The weights of a ring GEMM: W (K rows, zero rows up to Kp; N columns) in Nt-wide tiles.  `prebuilt`, if not null, is its image in
// the current split's format (an fp16x2 image carries its bf16x3 twin behind it); otherwise the images are built into img2 / img3.
// These may alias: the rerun builds its image after the fp16x2 launch, that image's last reader, has run.
struct RingWeights {
    int K, Kp, N, Nt;
    const float* W;
    uint8_t* img2;
    uint8_t* img3;
    const uint8_t* prebuilt = nullptr;
};
// The image of a launch with np pieces: the prebuilt one, or built from W into the workspace (img2 / img3).  A rerun (`run_if`, its
// flag, non-null) takes bf16x3 from the twin behind a prebuilt fp16x2 image, or builds it into img3 only if *run_if != 0.
inline int ring_image(const RingWeights& w, int np, const unsigned int* run_if, cudaStream_t st, const uint8_t*& image) {
    if (w.prebuilt != nullptr) {
        image = run_if != nullptr ? w.prebuilt + tc::tc_image_alloc_bytes(w.Kp, w.N, 2) : w.prebuilt;
        return PSA_OK;
    }
    uint8_t* own = np == 2 ? w.img2 : w.img3;
    image = own;
    return build_image(w.K, w.Kp, w.N, w.Nt | tc::image_flag(np), w.W, own, st, run_if);
}

// an output the kernel max-pools by ordered-int atomicMax: filled with the code of -inf before every launch, decoded after it
struct RingPool {
    float* out = nullptr;
    long long count = 0;
};

template <class Args>
int ring_launch_pooled(const RingKernels& k, int np, const Args& a, long long units, int Nt, const RingPool& pool, cudaStream_t st) {
    int rc;
    if (pool.out != nullptr && (rc = launch_fill_ord_neg_inf(pool.count, pool.out, st, a.ring.run_if)) != PSA_OK) return rc;
    if ((rc = ring_launch(k, np, Nt, &a, units, st)) != PSA_OK || pool.out == nullptr) return rc;
    return launch_decode_ord(pool.count, pool.out, st, a.ring.run_if);
}

// The bf16x3 rerun of an fp16x2 launch: its image build and its launch are no-ops unless the launch raised the word at `flag`.
// counter: null, or a zeroed word the rerun claims units from.  `a.ring` is filled in here.
template <class Args>
int ring_rerun(const RingKernels& k, Args a, long long units, const RingWeights& w, const unsigned int* flag, unsigned int* counter,
               cudaStream_t st, const RingPool& pool = {}) {
    const uint8_t* img3;
    const int rc = ring_image(w, 3, flag, st, img3);
    if (rc != PSA_OK) return rc;
    a.ring = RingArgs{};
    a.ring.image = img3; a.ring.run_if = flag; a.ring.counter = counter;
    return ring_launch_pooled(k, 3, a, units, w.Nt, pool, st);
}

// The op's ring GEMM in the current arithmetic mode.  Mode 2: bf16x3 only.  Otherwise the fp16x2 launch, which raises the zeroed
// word at `flag` when its result is invalid, then ring_rerun.  counters: null, or two zeroed words the launch and its rerun claim
// units from.  `a.ring` is filled in here.
template <class Args>
int ring_run(const RingKernels& k, Args a, long long units, const RingWeights& w, unsigned int* flag, unsigned int* counters,
             cudaStream_t st, const RingPool& pool = {}) {
    const int np = tc_np();
    const uint8_t* image;
    int rc = ring_image(w, np, nullptr, st, image);
    if (rc != PSA_OK) return rc;
    a.ring = RingArgs{};
    a.ring.image = image; a.ring.counter = counters;
    if (np == 3) return ring_launch_pooled(k, 3, a, units, w.Nt, pool, st);
    a.ring.ovf = flag; a.ring.wflag = image_trailer(image, w.Kp, w.N); a.ring.colscale = image_colscale(image, w.Kp, w.N);
    if ((rc = ring_launch_pooled(k, 2, a, units, w.Nt, pool, st)) != PSA_OK) return rc;
    return ring_rerun(k, a, units, w, flag, counters != nullptr ? counters + 1 : nullptr, st, pool);
}

}  // namespace psa
