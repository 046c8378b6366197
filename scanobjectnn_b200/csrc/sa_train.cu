// sa_train.cu -- training-mode front of a set-abstraction level ("variant F1", SURVEY 7 hard part 4).
//
// In training the reference's relu(BN(conv(x)+b)) needs batch statistics over all B*m*K rows before the ReLU
// (pointnet2/utils/tf_util.py:512-531, is_training=True), so the first 1x1 conv's PRE-BN output has to exist in HBM
// once.  The reference gets there through query_ball_point -> group_point -> tile/sub -> concat -> cuDNN conv + bias_add:
// four materialised (B,m,K,.) tensors.  This kernel does the whole front in ONE launch:
//   ball query (index-exact; exhaustive register search in the streaming kernel) -> neighbour coordinates from the shared-memory copy of
//   the cloud -> centre -> conv1 (+ optional per-point feature products U = points . W1[3:,:]) + bias ->
//   coalesced streaming store of (B,m,K,C1) + idx/pts_cnt + per-channel sum / sum-of-squares for the BN statistics.
// HBM traffic = algorithmic traffic: B*(12n + 12m) in, 4*B*m*K*(C1+1) + 4*B*m out  (137.3 MB at B=32,N=2048,m=512,K=32,
// C1=64) -- a pure write-bound kernel, the one BASELINE.json's ">= 70 % of the HBM roofline" target is defined on.
// Two kernels: the streaming kernel below whenever f1s_plan accepts the shape (n <= 4096, nsample <= 128, <= 110 KB of
// shared memory), the round-1 kernel sa_conv1_prebn_kernel (+ f1_stats_reduce_kernel for the statistics) otherwise.
#include <atomic>

#include "ball_query.cuh"
#include "common.cuh"

namespace psa {

float ball_query_threshold(float radius, bool* none);   // grouping.cu

constexpr int kF1Warps = kBqWarps;

struct F1Args {
    int n, m, nsample, C1, q_per_cta;
    float radius, thr;
    int none, want_grid;
    const float* xyz;      // (b,n,3)
    const float* new_xyz;  // (b,m,3)
    const float* uf;       // (b*n, C1) or null
    const float* w1;       // (3+c, C1): rows 0..2 used here
    const float* bias;     // (C1) or null
    float* pre;            // (b,m,K,C1)
    int* idx;              // (b,m,K)
    int* pts_cnt;          // (b,m) or null
    float* partial;        // (gridDim.x*gridDim.y, 2, C1) or null
};

// conv stage mapping: 8 lanes per row, 4 rows per warp step; lane-in-row s owns channels [32*i + 4*s, +4), i < NV = C1/32,
// so every store instruction writes 128 contiguous bytes per row and a query's K rows take K/4 steps.
template <int NV, bool STATS, int PPT>
__global__ void __launch_bounds__(kF1Warps * 32, PPT <= 8 ? 3 : 2)
sa_conv1_prebn_kernel(const __grid_constant__ F1Args a) {
    extern __shared__ __align__(16) float smem_f[];
    const int n = a.n;
    const int cloud = blockIdx.y;
    const float* gx = a.xyz + (size_t)cloud * n * 3;       // neighbour coordinates come from global memory / L1 (24 KB per cloud)
    const BqSmem s = bq_carve(smem_f, n, a.want_grid != 0, gx);
    int* srow = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(smem_f) + bq_smem_bytes(n, a.want_grid != 0));   // kF1Warps * nsample
    float* sstat = reinterpret_cast<float*>(srow + kF1Warps * ((a.nsample + 3) & ~3));   // kF1Warps * 2 * C1 (STATS), 16-B aligned
    const BqGrid g = bq_stage_and_build<PPT>(s, n, a.radius, a.want_grid != 0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & 7, rsub = lane >> 3;
    // float pairs: pair p of vector i covers channels 32*i + 4*sub + 2*p, +1
    constexpr int NPK = 2 * NV;
    float2 wx[NPK], wy[NPK], wz[NPK], bs[NPK], ssum[NPK], ssq[NPK];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = 32 * i + 4 * sub;
        const float4 x4 = __ldg(reinterpret_cast<const float4*>(a.w1 + c));
        const float4 y4 = __ldg(reinterpret_cast<const float4*>(a.w1 + a.C1 + c));
        const float4 z4 = __ldg(reinterpret_cast<const float4*>(a.w1 + 2 * a.C1 + c));
        const float4 b4 = a.bias ? __ldg(reinterpret_cast<const float4*>(a.bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
        wx[2 * i] = make_float2(x4.x, x4.y); wx[2 * i + 1] = make_float2(x4.z, x4.w);
        wy[2 * i] = make_float2(y4.x, y4.y); wy[2 * i + 1] = make_float2(y4.z, y4.w);
        wz[2 * i] = make_float2(z4.x, z4.y); wz[2 * i + 1] = make_float2(z4.z, z4.w);
        bs[2 * i] = make_float2(b4.x, b4.y); bs[2 * i + 1] = make_float2(b4.z, b4.w);
        ssum[2 * i] = ssum[2 * i + 1] = make_float2(0.f, 0.f);
        ssq[2 * i] = ssq[2 * i + 1] = make_float2(0.f, 0.f);
    }
    const int q0 = blockIdx.x * a.q_per_cta;
    const int q1 = min(a.m, q0 + a.q_per_cta);
    const float* p2 = a.new_xyz + (size_t)cloud * a.m * 3;
    int* row = srow + warp * a.nsample;
    const float* ucloud = a.uf ? a.uf + (size_t)cloud * n * a.C1 + 4 * sub : nullptr;
    for (int q = q0 + warp; q < q1; q += kF1Warps) {
        const float qx = __ldg(p2 + q * 3 + 0), qy = __ldg(p2 + q * 3 + 1), qz = __ldg(p2 + q * 3 + 2);
        const int cnt = bq_query_warp(n, a.nsample, a.thr, a.none != 0, s, g, qx, qy, qz, row, lane, warp);
        __syncwarp();
        const size_t gq = (size_t)cloud * a.m + q;
        for (int l = lane; l < a.nsample; l += 32) a.idx[gq * a.nsample + l] = row[l];
        if (a.pts_cnt != nullptr && lane == 0) a.pts_cnt[gq] = cnt;
        float* outl = a.pre + gq * a.nsample * a.C1 + 4 * sub;          // this lane's column offset inside the query's block
        for (int r0 = 0; r0 < a.nsample; r0 += 4) {
            const int r = r0 + rsub;
            if (r < a.nsample) {
                const int j = row[r];
                // grouped_xyz - new_xyz (pointnet_util.py:46), broadcast into both halves of a packed register
                const float dxs = __ldg(gx + 3 * j) - qx, dys = __ldg(gx + 3 * j + 1) - qy, dzs = __ldg(gx + 3 * j + 2) - qz;
                const float2 dx = make_float2(dxs, dxs), dy = make_float2(dys, dys), dz = make_float2(dzs, dzs);
                const float* urow = ucloud ? ucloud + (unsigned)j * (unsigned)a.C1 : nullptr;
                float* orow = outl + (unsigned)r * (unsigned)a.C1;
#pragma unroll
                for (int i = 0; i < NV; ++i) {
                    float2 s0 = bs[2 * i], s1 = bs[2 * i + 1];
                    if (urow) {
                        const float4 u = __ldg(reinterpret_cast<const float4*>(urow + 32 * i));
                        s0 = fadd2_rn(s0, make_float2(u.x, u.y)); s1 = fadd2_rn(s1, make_float2(u.z, u.w));
                    }
                    // two channels per float pair
                    const float2 v0 = ffma2_rn(dz, wz[2 * i], ffma2_rn(dy, wy[2 * i], ffma2_rn(dx, wx[2 * i], s0)));
                    const float2 v1 = ffma2_rn(dz, wz[2 * i + 1], ffma2_rn(dy, wy[2 * i + 1], ffma2_rn(dx, wx[2 * i + 1], s1)));
                    __stcs(reinterpret_cast<float4*>(orow + 32 * i), make_float4(v0.x, v0.y, v1.x, v1.y));   // streaming store
                    if (STATS) {
                        ssum[2 * i] = fadd2_rn(ssum[2 * i], v0); ssum[2 * i + 1] = fadd2_rn(ssum[2 * i + 1], v1);
                        ssq[2 * i] = ffma2_rn(v0, v0, ssq[2 * i]); ssq[2 * i + 1] = ffma2_rn(v1, v1, ssq[2 * i + 1]);
                    }
                }
            }
        }
        __syncwarp();
    }
    if (STATS) {
        // the four row-groups of a warp hold partials of the same channels: fold them, then one row-group publishes
#pragma unroll
        for (int p = 0; p < NPK; ++p) {
#pragma unroll
            for (int o = 8; o < 32; o <<= 1) {
                ssum[p].x += __shfl_xor_sync(0xffffffffu, ssum[p].x, o); ssum[p].y += __shfl_xor_sync(0xffffffffu, ssum[p].y, o);
                ssq[p].x += __shfl_xor_sync(0xffffffffu, ssq[p].x, o); ssq[p].y += __shfl_xor_sync(0xffffffffu, ssq[p].y, o);
            }
            if (rsub == 0) {
                float* w = sstat + (size_t)warp * 2 * a.C1;
                const int c = 32 * (p >> 1) + 4 * sub + 2 * (p & 1);
                *reinterpret_cast<float2*>(w + c) = ssum[p];
                *reinterpret_cast<float2*>(w + a.C1 + c) = ssq[p];
            }
        }
        __syncthreads();
        float* dst = a.partial + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 2 * a.C1;
        for (int e = threadIdx.x; e < 2 * a.C1; e += blockDim.x) {
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < kF1Warps; ++w) t += sstat[(size_t)w * 2 * a.C1 + e];   // fixed order: deterministic
            dst[e] = t;
        }
    }
}


// ---------------------------------------------------------------------------------------------------------------------
// Streaming F1 kernel (round 2, wherever f1s_plan fits): the same front as above, organised so that the only thing the SMs do for most of
// the launch is stream the (B,m,K,C1) tensor out.
//   * persistent CTAs (2 per SM, 12 warps), each owning a contiguous range of the B*m queries; when the grid is a multiple of
//     B every CTA stays inside one cloud (ranges that cross a cloud boundary reload the cloud and re-ramp the pipeline);
//   * three warpgroups = three pipeline stages (registers re-partitioned with setmaxnreg: 128 / 56 / 56):
//       SEARCH   warps 0-3.  No spatial grid: at these sizes (n <= 4096, ~60 queries per CTA) an exhaustive test out of
//                REGISTERS is cheaper than building one.  A search thread keeps PPTP CONSECUTIVE points of the cloud in
//                registers as float pairs and tests them against every query of a batch with the reference's
//                arithmetic (NaN counts as inside); the SIGN of (thr - d) is shifted straight into the lane's hit mask, and
//                because the lane's points are consecutive that mask IS bits [PPTP*tid, +PPTP) of the query's bitmap -- no
//                ballots, no atomics, no compaction;
//       EXTRACT  warps 4-7.  LPQ = 16 lanes per query read the nsample lowest set bits out in index order (popcount prefix
//                sums: the reference's "first nsample in index order", padded with the first hit), write idx / pts_cnt to
//                global memory and the centred rows (dx,dy,dz,j) of the batch into the rows ring;
//       CONV     warps 8-11.  Per step 4 rows x C1 channels -- one LDS.128 for the row's (dx,dy,dz,j), 12 FFMA per 4 channels
//                with the weights resident in registers, 128-byte streaming stores, BN statistics in registers.
//     Levels WITH input features (HAS_U) run two stages instead: warps 0-3 search and extract, warps 4-11 convolve (the
//     512-byte U-row gathers of the conv stage are what needs the warps there);
//   * two rings of kF1Ring slots (bitmaps + centres | rows), named barriers FULL/EMPTY per slot; batches of 2, 4, then
//     kF1Batch queries so the first stores leave early.  No CTA-wide barrier inside the main loop.
// Statistics: per-CTA partials in a fixed order, the last CTA to finish (ticket) adds them in fp64 in CTA order:
// deterministic, one launch.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kF1WThreads = 384;           // streaming kernel: one warpgroup of search warps + two of worker warps
constexpr int kF1NP = 4;
constexpr int kF1Batch = 8;                // smallest full batch (two queries per worker warp, four worker warps): sizes the grid
constexpr int kF1Ring = 3;                 // bitmap slots in flight (5 / 6 measured: no change -- the search warps never run ahead)
constexpr int kF1Tickets = 64;

// completion tickets of the statistics reduction: zero at load, reset by the last CTA of every launch; a launch uses
// ticket (call number mod 64), so up to 64 launches may be in flight at once (different streams / CUDA graphs)
__device__ unsigned g_f1_tickets[kF1Tickets];

struct F1SArgs {
    int b, n, m, nsample, C1;
    float thr;
    int none;
    const float* xyz;
    const float* new_xyz;
    const float* uf;
    const float* w1;
    const float* bias;
    float* pre;
    int* idx;
    int* pts_cnt;
    float* partial;        // (gridDim.x, 2, C1)
    float* stats;          // (2, C1) or null
    int ticket;            // index into g_f1_tickets
};

__device__ __forceinline__ void named_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// Batches of a cloud segment: 2, 4, then kF1Batch queries -- the first stores of a CTA start after a 2-query search.
__host__ __device__ inline int f1s_batch_size(int t, int qb) { return t == 0 ? 2 : (t == 1 ? 4 : qb); }
__host__ __device__ inline int f1s_num_batches(long long nq, int qb) {
    int t = 0;
    for (long long done = 0; done < nq; ++t) done += f1s_batch_size(t, qb);
    return t;
}

// shared memory: cloud as float4 (x,y,z,bits(k)) | kF1Batch bitmaps of bw words | ring slots (idx rows | centred rows)
__host__ __device__ inline int f1s_bitmap_words(int np, int pptp) { const int w = np * pptp; return w < 32 ? 32 : w; }
__host__ __device__ inline size_t f1s_smem_bytes(int n, int nsample, int np, int pptp) {
    // cloud copy | ring B: bitmaps + centres | ring R: idx rows + centred rows (reused by the statistics epilogue: up to 12 KB of partials)
    size_t ringb = (size_t)kF1Ring * kF1Batch * (f1s_bitmap_words(np, pptp) * 4 + sizeof(float4));
    size_t ringr = (size_t)kF1Ring * kF1Batch * nsample * (sizeof(int) + sizeof(float4));
    if (ringr < 12288) ringr = 12288;
    return (size_t)n * 16 + ringb + ringr;
}

// float pairs in 64-bit registers, each half rounded on its own (sm_90 has no packed f32x2 instructions: two scalar ops each)
typedef unsigned long long u64;
__device__ __forceinline__ u64 f2_pack(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ float2 f2_split(u64 v) { float lo, hi; asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); return make_float2(lo, hi); }
__device__ __forceinline__ u64 f2_add(u64 a, u64 b) { const float2 x = f2_split(a), y = f2_split(b); return f2_pack(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y)); }
__device__ __forceinline__ u64 f2_sub(u64 a, u64 b) { const float2 x = f2_split(a), y = f2_split(b); return f2_pack(__fsub_rn(x.x, y.x), __fsub_rn(x.y, y.y)); }
__device__ __forceinline__ u64 f2_mul(u64 a, u64 b) { const float2 x = f2_split(a), y = f2_split(b); return f2_pack(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y)); }
__device__ __forceinline__ u64 f2_fma(u64 a, u64 b, u64 c) {
    const float2 x = f2_split(a), y = f2_split(b), z = f2_split(c);
    return f2_pack(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}
__device__ __forceinline__ void f2_unpack_bits(u64 v, unsigned& lo, unsigned& hi) { asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v)); }

template <int NV, bool HAS_U, int PPTP>
__global__ void __launch_bounds__(kF1WThreads, 2)       // 80 registers at launch; setmaxnreg: search warps 128, the others 56
sa_conv1_stream_kernel(const __grid_constant__ F1SArgs a) {
    // three pipelined stages, one warpgroup each (measured on the two-stage kernel: search 24 k, extraction + rows 18 k, conv + store 18 k
    // cycles per CTA -- in series on the producer warps they set the kernel time, side by side the slowest one does):
    //   warps 0-3  SEARCH : the cloud in registers, exhaustive packed-f32x2 test -> hit bitmaps            (ring B: bitmaps, centres)
    //   warps 4-7  EXTRACT: bitmap -> nsample first hits in index order (idx, pts_cnt) -> centred rows     (ring R: rows)
    //   warps 8-11 CONV   : rows -> conv1 + bias (+ U) -> 512-byte streaming stores, BN statistics in registers
    constexpr int NP = kF1NP;                              // warps per stage
    constexpr int QB = kF1Batch;                           // queries per batch
    constexpr bool TWO = HAS_U;                            // levels with input features: two stages -- warps 0-3 search AND extract, warps 4-11 conv + store
                                                           // (the U-row gather of the conv stage is what needs the warps there: 64 vs 83 us at SA2)
    constexpr int CONV0 = TWO ? NP : 2 * NP;               // first conv warp
    constexpr int NC = kF1WThreads / 32 - CONV0;           // conv warps: 4 or 8
    constexpr int RCNT = TWO ? kF1WThreads : 2 * NP * 32;  // threads on the ring-R barriers
    constexpr int PT = NP * 32;                            // threads per stage
    constexpr int BW = NP * PPTP < 32 ? 32 : NP * PPTP;    // bitmap words per query
    constexpr int C1c = NV * 32;                           // = a.C1 (the launcher picks NV = C1 / 32)
    constexpr int LPQ = 32 * NP / QB;                      // lanes per query in the extraction: 16
    constexpr int BAR_BFULL = 1, BAR_BEMPTY = 1 + kF1Ring, BAR_RFULL = 1 + 2 * kF1Ring, BAR_REMPTY = 1 + 3 * kF1Ring, BAR_CLOUD = 1 + 4 * kF1Ring;
    static_assert(BAR_CLOUD <= 15, "named barriers");
    extern __shared__ __align__(16) float smem_f[];
    const int n = a.n, K = a.nsample, C1 = a.C1;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float4* cloud4 = reinterpret_cast<float4*>(smem_f);
    unsigned* bitmaps = reinterpret_cast<unsigned*>(cloud4 + n);                                  // kF1Ring x QB x BW
    float4* centres = reinterpret_cast<float4*>(bitmaps + kF1Ring * QB * BW);                     // kF1Ring x QB
    uint8_t* ring = reinterpret_cast<uint8_t*>(centres + kF1Ring * QB);                           // ring R; reused by the statistics epilogue
    const size_t slot_bytes = (size_t)QB * K * (sizeof(int) + sizeof(float4));                    // idx rows | centred rows
    __shared__ int4 s_hdrB[kF1Ring];                       // (first query - q_begin, queries [0 = stop], last batch of a cloud with more to come, -)
    __shared__ int2 s_hdrR[kF1Ring];                       // (first query - q_begin, queries [0 = stop])

    float2 ssum[2], ssq[2];                                // this lane's four channels (conv warps)
    ssum[0] = ssum[1] = ssq[0] = ssq[1] = make_float2(0.f, 0.f);

    const long long T = (long long)a.b * a.m;
    // a grid that is a multiple of the batch size gives every cloud the same number of CTAs: no CTA crosses a cloud boundary (a
    // crossing costs a second cloud load + pipeline ramp)
    long long q_begin, q_end;
    if (gridDim.x % a.b == 0) {
        const int cpc = gridDim.x / a.b, cl = blockIdx.x / cpc, ci = blockIdx.x % cpc;
        q_begin = (long long)cl * a.m + (long long)a.m * ci / cpc;
        q_end = (long long)cl * a.m + (long long)a.m * (ci + 1) / cpc;
    } else {
        q_begin = T * blockIdx.x / gridDim.x; q_end = T * (blockIdx.x + 1) / gridDim.x;
    }

    // bitmap -> the query's nsample first hits in index order (idx, pts_cnt) -> centred rows grouped_xyz - new_xyz (pointnet_util.py:46)
    // + the source index for the U gather, into ring-R slot `slot`; LPQ lanes per query, executed by the PT threads of one stage
    // (w, t = warp / thread index inside that stage); `release` runs once the bitmaps and centres have been read
    auto extract_rows = [&](const int slot, const unsigned* bmq, const float4* ctrq, const long long gq0, const int nqb, const int w, auto release) {
        int* sidx = reinterpret_cast<int*>(ring + slot * slot_bytes);
        float4* sd = reinterpret_cast<float4*>(ring + slot * slot_bytes + (size_t)QB * K * sizeof(int));
        const int qi = w * (32 / LPQ) + lane / LPQ, sub = lane & (LPQ - 1);
        const bool act = qi < nqb;
        const int cnt = bq_extract_bitmap_sub<LPQ, BW / LPQ>(bmq + (size_t)qi * BW, K, sidx + qi * K, lane, act);
        const float4 ctr = act ? ctrq[qi] : make_float4(0.f, 0.f, 0.f, 0.f);
        __syncwarp();                                                                       // the query's idx row is complete (one warp)
        release();
        if (act) {
            if (a.pts_cnt != nullptr && sub == 0) a.pts_cnt[gq0 + qi] = cnt;
            int* gidx = a.idx + (size_t)(gq0 + qi) * K;
            for (int r = sub; r < K; r += LPQ) {
                const int j = sidx[qi * K + r];
                const float4 pt = cloud4[j];
                gidx[r] = j;
                sd[qi * K + r] = make_float4(pt.x - ctr.x, pt.y - ctr.y, pt.z - ctr.z, __int_as_float(j));
            }
        }
    };

    if (warp < NP) {
        // =========================================== SEARCH (+ EXTRACT when TWO) ===========================================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 128;");               // the cloud lives in registers
        for (int i = tid; i < kF1Ring * QB * BW; i += PT) bitmaps[i] = 0u;   // words no warp owns (BW > NP*PPTP) stay zero
        int ring_pos = 0;
        bool first_cloud = true;
        for (long long q = q_begin; q < q_end;) {
            const long long cloud = q / a.m;
            const long long seg_end = min(q_end, (cloud + 1) * (long long)a.m);
            const float* gx = a.xyz + (size_t)cloud * n * 3;
            // first batch's query centres: in flight together with the cloud (lane i of every search warp holds query i of a batch)
            long long gq0 = q;                                                             // global query id of the batch
            float ncx = 0.f, ncy = 0.f, ncz = 0.f;
            if (lane < min(f1s_batch_size(0, QB), (int)(seg_end - gq0))) {
                const float* p2 = a.new_xyz + (size_t)(gq0 + lane) * 3;
                ncx = __ldg(p2); ncy = __ldg(p2 + 1); ncz = __ldg(p2 + 2);
            }
            // ---- this cloud: PPTP CONSECUTIVE points per thread in registers (point k = PPTP*(32*warp + lane) + i) as packed
            //      f32x2 pairs (points 2j, 2j+1), so the lane's hit mask IS bits [PPTP*(32*warp+lane), +PPTP) of the query's
            //      bitmap -- no ballots, no transposition; float4 copy of the cloud in shared memory for the row builder ----
            if (!first_cloud) {                                              // the extraction no longer reads the previous cloud's copy
                if (TWO) named_bar_sync(15, PT); else named_bar_sync(BAR_CLOUD, 2 * PT);
            }
            first_cloud = false;
            u64 px[PPTP / 2], py[PPTP / 2], pz[PPTP / 2];
            unsigned valid = 0u;
            const int k0 = PPTP * tid;                                       // tid = 32 * warp + lane < PT
            if (((n & 3) | (int)(reinterpret_cast<uintptr_t>(a.xyz) & 15)) == 0) {
                // one round trip: the lane's PPTP points are 3*PPTP/4 consecutive float4 (16-byte aligned: n % 4 == 0), all loads in
                // flight at once; registers and the shared-memory copy are both filled from them
                constexpr int CH = PPTP == 32 ? 2 : 1;                       // 32 points per thread: two halves of 12 float4
                constexpr int PH = PPTP / CH;
                const float4* g4 = reinterpret_cast<const float4*>(gx);
                const int nf4 = n * 3 / 4;
#pragma unroll
                for (int hh = 0; hh < CH; ++hh) {
                    float f[3 * PH];
#pragma unroll
                    for (int v = 0; v < 3 * PH / 4; ++v) {
                        const int fi = (k0 + hh * PH) * 3 / 4 + v;
                        const float4 t = fi < nf4 ? __ldg(g4 + fi) : make_float4(0.f, 0.f, 0.f, 0.f);
                        f[4 * v] = t.x; f[4 * v + 1] = t.y; f[4 * v + 2] = t.z; f[4 * v + 3] = t.w;
                    }
#pragma unroll
                    for (int i = 0; i < PH; ++i) {
                        const int k = k0 + hh * PH + i;
                        if (k < n) { valid |= 1u << (hh * PH + i); cloud4[k] = make_float4(f[3 * i], f[3 * i + 1], f[3 * i + 2], __int_as_float(k)); }
                    }
#pragma unroll
                    for (int j = 0; j < PH / 2; ++j) {
                        px[hh * PH / 2 + j] = f2_pack(f[6 * j], f[6 * j + 3]);
                        py[hh * PH / 2 + j] = f2_pack(f[6 * j + 1], f[6 * j + 4]);
                        pz[hh * PH / 2 + j] = f2_pack(f[6 * j + 2], f[6 * j + 5]);
                    }
                }
            } else {
                for (int k = tid; k < n; k += PT)
                    cloud4[k] = make_float4(__ldg(gx + 3 * k), __ldg(gx + 3 * k + 1), __ldg(gx + 3 * k + 2), __int_as_float(k));
#pragma unroll
                for (int j = 0; j < PPTP / 2; ++j) {
                    float c[6];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int k = k0 + 2 * j + h;
                        c[3 * h] = c[3 * h + 1] = c[3 * h + 2] = 0.f;       // slots past the cloud: masked out by `valid`
                        if (k < n) {
                            c[3 * h] = __ldg(gx + 3 * k); c[3 * h + 1] = __ldg(gx + 3 * k + 1); c[3 * h + 2] = __ldg(gx + 3 * k + 2);
                            valid |= 1u << (2 * j + h);
                        }
                    }
                    px[j] = f2_pack(c[0], c[3]); py[j] = f2_pack(c[1], c[4]); pz[j] = f2_pack(c[2], c[5]);
                }
            }
            const u64 thr2 = f2_pack(a.thr, a.thr);
            // the NEXT batch's centres are fetched under the current search
            for (int bi = 0; gq0 < seg_end; ++bi, ++ring_pos) {
                const int slot = ring_pos % kF1Ring;
                const int nqb = min(f1s_batch_size(bi, QB), (int)(seg_end - gq0));
                const int bslot = TWO ? (ring_pos & 1) : slot;                              // TWO: bitmaps double-buffered inside the stage
                unsigned* bms = bitmaps + (size_t)bslot * QB * BW;
                const float cqx = ncx, cqy = ncy, cqz = ncz;
                {
                    const long long gq1 = gq0 + nqb;
                    if (gq1 < seg_end && lane < min(f1s_batch_size(bi + 1, QB), (int)(seg_end - gq1))) {
                        const float* p2 = a.new_xyz + (size_t)(gq1 + lane) * 3;
                        ncx = __ldg(p2); ncy = __ldg(p2 + 1); ncz = __ldg(p2 + 2);
                    }
                }
                if (!TWO && ring_pos >= kF1Ring) named_bar_sync(BAR_BEMPTY + slot, 2 * PT); // slot drained by the extraction
                if (warp == 0 && lane < nqb) centres[bslot * QB + lane] = make_float4(cqx, cqy, cqz, 0.f);
                if (!TWO && tid == 0) s_hdrB[slot] = make_int4((int)(gq0 - q_begin), nqb, (gq0 + nqb == seg_end && seg_end < q_end) ? 1 : 0, 0);
                // ---- exhaustive test on float pairs: per point 3 FADD + FMUL + 2 FFMA (the reference's
                //      distance) + one FADD s = thr - d + funnel shifts that push the SIGN of s into the lane's mask.
                //      sign(s) = 1 <=> d > thr; d == thr gives +0 and a NaN distance the canonical (positive) NaN, i.e. both
                //      count as inside exactly like !(d > thr) (tf_grouping_g.cu:20-21: max(sqrtf(NaN),1e-20f) < r holds) ----
                if (!a.none) {
                    for (int qi = 0; qi < nqb; ++qi) {
                        const float qx = __shfl_sync(0xffffffffu, cqx, qi), qy = __shfl_sync(0xffffffffu, cqy, qi), qz = __shfl_sync(0xffffffffu, cqz, qi);
                        const u64 nqx = f2_pack(-qx, -qx), nqy = f2_pack(-qy, -qy), nqz = f2_pack(-qz, -qz);
                        unsigned acc[PPTP / 8];                              // 8 points per chain: short dependency chains
#pragma unroll
                        for (int g = 0; g < PPTP / 8; ++g) acc[g] = 0u;
#pragma unroll
                        for (int j = PPTP / 2 - 1; j >= 0; --j) {            // descending: point i ends up at bit i of its chain
                            const u64 dx = f2_add(px[j], nqx), dy = f2_add(py[j], nqy), dz = f2_add(pz[j], nqz);
                            u64 t = f2_mul(dy, dy);
                            t = f2_fma(dx, dx, t);
                            t = f2_fma(dz, dz, t);
                            unsigned slo, shi;
                            f2_unpack_bits(f2_sub(thr2, t), slo, shi);
                            acc[j >> 2] = __funnelshift_l(shi, acc[j >> 2], 1);
                            acc[j >> 2] = __funnelshift_l(slo, acc[j >> 2], 1);
                        }
                        unsigned outside = acc[0];
#pragma unroll
                        for (int g = 1; g < PPTP / 8; ++g) outside |= acc[g] << (8 * g);
                        const unsigned inside = ~outside & valid;
                        uint8_t* bm = reinterpret_cast<uint8_t*>(bms + qi * BW) + (32 * warp + lane) * (PPTP / 8);
                        if (PPTP == 8) *bm = (uint8_t)inside;
                        else if (PPTP == 16) *reinterpret_cast<unsigned short*>(bm) = (unsigned short)inside;
                        else *reinterpret_cast<unsigned*>(bm) = inside;
                    }
                }
                if (TWO) {
                    named_bar_sync(15, PT);                                                 // bitmaps + centres (+ the cloud copy) complete
                    if (ring_pos >= kF1Ring) named_bar_sync(BAR_REMPTY + slot, RCNT);       // rows slot drained by the conv warps
                    extract_rows(slot, bms, centres + bslot * QB, gq0, nqb, warp, [] {});
                    if (tid == 0) s_hdrR[slot] = make_int2((int)(gq0 - q_begin), nqb);
                    __threadfence_block();
                    named_bar_arrive(BAR_RFULL + slot, RCNT);
                } else {
                    __threadfence_block();
                    named_bar_arrive(BAR_BFULL + slot, 2 * PT);                             // bitmaps + centres (+ the cloud copy) ready
                }
                gq0 += nqb;
            }
            q = seg_end;
        }
        // stop marker, then take the next stage's outstanding releases (every arrival has a taker: no barrier is left half full)
        {
            const int slot = ring_pos % kF1Ring;
            if (TWO) {
                if (ring_pos >= kF1Ring) named_bar_sync(BAR_REMPTY + slot, RCNT);
                if (tid == 0) s_hdrR[slot] = make_int2(0, 0);
                __threadfence_block();
                named_bar_arrive(BAR_RFULL + slot, RCNT);
                for (int p = ring_pos + 1; p <= ring_pos + kF1Ring; ++p)
                    if (p >= kF1Ring) named_bar_sync(BAR_REMPTY + p % kF1Ring, RCNT);
            } else {
                if (ring_pos >= kF1Ring) named_bar_sync(BAR_BEMPTY + slot, 2 * PT);
                if (tid == 0) s_hdrB[slot] = make_int4(0, 0, 0, 0);
                __threadfence_block();
                named_bar_arrive(BAR_BFULL + slot, 2 * PT);
                for (int p = ring_pos + 1; p <= ring_pos + kF1Ring; ++p)
                    if (p >= kF1Ring) named_bar_sync(BAR_BEMPTY + p % kF1Ring, 2 * PT);
            }
        }
    } else if (!TWO && warp < 2 * NP) {
        // =========================================== EXTRACT ===========================================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int ew = warp - NP, et = tid - PT;
        for (int ring_pos = 0;; ++ring_pos) {
            const int slot = ring_pos % kF1Ring;
            named_bar_sync(BAR_BFULL + slot, 2 * PT);
            const int4 hdr = s_hdrB[slot];
            const int nqb = hdr.y;
            if (ring_pos >= kF1Ring) named_bar_sync(BAR_REMPTY + slot, RCNT);               // rows slot drained by the conv warps
            if (nqb == 0) {                                                                 // stop: pass it on, take the outstanding releases
                named_bar_arrive(BAR_BEMPTY + slot, 2 * PT);
                if (et == 0) s_hdrR[slot] = make_int2(0, 0);
                __threadfence_block();
                named_bar_arrive(BAR_RFULL + slot, RCNT);
                for (int p = ring_pos + 1; p <= ring_pos + kF1Ring; ++p)
                    if (p >= kF1Ring) named_bar_sync(BAR_REMPTY + p % kF1Ring, RCNT);
                break;
            }
            extract_rows(slot, bitmaps + (size_t)slot * QB * BW, centres + slot * QB, q_begin + hdr.x, nqb, ew,
                         [&] { named_bar_arrive(BAR_BEMPTY + slot, 2 * PT); });             // bitmaps + centres consumed
            if (et == 0) s_hdrR[slot] = make_int2(hdr.x, nqb);
            __threadfence_block();
            named_bar_arrive(BAR_RFULL + slot, RCNT);
            if (hdr.z) named_bar_arrive(BAR_CLOUD, 2 * PT);                                 // last batch of this cloud: its copy is free
        }
    } else {
        // =========================================== CONV + STORE ===========================================
        // lane mapping: LPR = C1/4 lanes cover one row (4 consecutive channels each), so a warp store instruction writes
        // 32/LPR whole rows = 512 contiguous bytes; a lane's channels are fixed, its weights live in registers
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int cw = warp - CONV0;
        constexpr int LPR = NV * 8;                    // 16 (C1 = 64) or 32 (C1 = 128)
        constexpr int RPI = 32 / LPR;                  // rows per store instruction: 2 or 1
        const int lr = lane / LPR, lc = (lane % LPR) * 4;
        const float4 wx4 = __ldg(reinterpret_cast<const float4*>(a.w1 + lc));
        const float4 wy4 = __ldg(reinterpret_cast<const float4*>(a.w1 + C1 + lc));
        const float4 wz4 = __ldg(reinterpret_cast<const float4*>(a.w1 + 2 * C1 + lc));
        const float4 b4 = a.bias ? __ldg(reinterpret_cast<const float4*>(a.bias + lc)) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float2 wxa = make_float2(wx4.x, wx4.y), wxb = make_float2(wx4.z, wx4.w), wya = make_float2(wy4.x, wy4.y), wyb = make_float2(wy4.z, wy4.w);
        const float2 wza = make_float2(wz4.x, wz4.y), wzb = make_float2(wz4.z, wz4.w), ba = make_float2(b4.x, b4.y), bb = make_float2(b4.z, b4.w);
        for (int ring_pos = 0;; ++ring_pos) {
            const int slot = ring_pos % kF1Ring;
            const float4* sd = reinterpret_cast<const float4*>(ring + slot * slot_bytes + (size_t)QB * K * sizeof(int));
            named_bar_sync(BAR_RFULL + slot, RCNT);
            const int2 hdr = s_hdrR[slot];
            const int nqb = hdr.y;
            if (nqb == 0) { named_bar_arrive(BAR_REMPTY + slot, RCNT); break; }               // stop marker
            const long long gq0 = q_begin + hdr.x;
            const int nrows = nqb * K;
            float* outl = a.pre + (size_t)gq0 * K * C1c + lc;
            const float* ucloud = HAS_U ? a.uf + (size_t)(gq0 / a.m) * n * C1c + lc : nullptr;
            // four rows per lane and trip: independent chains, stores of a warp instruction contiguous; C1 is a compile-time
            // constant (immediate store offsets, one pointer bump per trip); row guards only when nrows is not a multiple of 4*RPI
            auto row = [&](const float4 d, float* dst) {
                float2 s0 = ba, s1 = bb;
                if (HAS_U) {
                    const float4 uu = __ldg(reinterpret_cast<const float4*>(ucloud + (unsigned)__float_as_int(d.w) * (unsigned)C1c));
                    s0 = fadd2_rn(s0, make_float2(uu.x, uu.y)); s1 = fadd2_rn(s1, make_float2(uu.z, uu.w));
                }
                const float2 dx = make_float2(d.x, d.x), dy = make_float2(d.y, d.y), dz = make_float2(d.z, d.z);
                const float2 v0 = ffma2_rn(dz, wza, ffma2_rn(dy, wya, ffma2_rn(dx, wxa, s0)));
                const float2 v1 = ffma2_rn(dz, wzb, ffma2_rn(dy, wyb, ffma2_rn(dx, wxb, s1)));
                __stcs(reinterpret_cast<float4*>(dst), make_float4(v0.x, v0.y, v1.x, v1.y));
                ssum[0] = fadd2_rn(ssum[0], v0); ssum[1] = fadd2_rn(ssum[1], v1);
                ssq[0] = ffma2_rn(v0, v0, ssq[0]); ssq[1] = ffma2_rn(v1, v1, ssq[1]);
            };
            if ((nrows & (4 * RPI - 1)) == 0) {
                const float4* sp = sd + cw * 4 * RPI + lr;
                float* op = outl + (size_t)(cw * 4 * RPI + lr) * C1c;
                for (int r0 = cw * 4 * RPI; r0 < nrows; r0 += NC * 4 * RPI, sp += NC * 4 * RPI, op += (size_t)NC * 4 * RPI * C1c) {
                    float4 d[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) d[u] = sp[u * RPI];
#pragma unroll
                    for (int u = 0; u < 4; ++u) row(d[u], op + u * RPI * C1c);
                }
            } else {
                for (int r0 = cw * 4 * RPI; r0 < nrows; r0 += NC * 4 * RPI) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int r = r0 + u * RPI + lr;
                        if (r < nrows) row(sd[r], outl + (size_t)r * C1c);
                    }
                }
            }
            named_bar_arrive(BAR_REMPTY + slot, RCNT);
        }
    }

    // back to the launch allocation (80 registers each) for the common epilogue
    if (warp < NP) asm volatile("setmaxnreg.dec.sync.aligned.u32 80;");
    else asm volatile("setmaxnreg.inc.sync.aligned.u32 80;");
    if (a.stats != nullptr) {
        __syncthreads();                                   // ring memory is free: reuse it for the per-warp partials
        float* sstat = reinterpret_cast<float*>(ring);     // NC x 2 x C1
        {
            constexpr int LPR = NV * 8;
            // lanes lr = 0 .. 32/LPR-1 of a warp hold partials of the same four channels: fold them, lane row 0 publishes
#pragma unroll
            for (int p = 0; p < 2; ++p) {
#pragma unroll
                for (int o = LPR; o < 32; o <<= 1) {
                    ssum[p].x += __shfl_xor_sync(0xffffffffu, ssum[p].x, o); ssum[p].y += __shfl_xor_sync(0xffffffffu, ssum[p].y, o);
                    ssq[p].x += __shfl_xor_sync(0xffffffffu, ssq[p].x, o); ssq[p].y += __shfl_xor_sync(0xffffffffu, ssq[p].y, o);
                }
                if (warp >= CONV0 && lane < LPR) {
                    float* w = sstat + (size_t)(warp - CONV0) * 2 * C1;
                    const int c = lane * 4 + 2 * p;
                    *reinterpret_cast<float2*>(w + c) = ssum[p];
                    *reinterpret_cast<float2*>(w + C1 + c) = ssq[p];
                }
            }
        }
        __syncthreads();
        float* dst = a.partial + (size_t)blockIdx.x * 2 * C1;
        for (int e = tid; e < 2 * C1; e += kF1WThreads) {
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < NC; ++w) t += sstat[(size_t)w * 2 * C1 + e];      // fixed order
            dst[e] = t;
        }
        // last CTA to arrive adds the CTA partials (fp64) in a fixed tree: deterministic whatever the finishing order
        __shared__ unsigned s_last;
        __threadfence();
        __syncthreads();
        if (tid == 0) s_last = (atomicAdd(&g_f1_tickets[a.ticket], 1u) == gridDim.x - 1) ? 1u : 0u;
        __syncthreads();
        if (s_last) {
            __threadfence();
            // thread (rl, e4): partial rows p = rl, rl + RL, ... of float4 column e4, sixteen loads in flight (the loop is
            // L2-latency-bound), fp64 accumulators in ascending p; then the RL row lanes in order through shared memory
            const int E4 = 2 * C1 / 4;                                     // 32 (C1 = 64) or 64 (C1 = 128)
            const int RL = kF1WThreads / E4;                               // 8 or 4
            const int e4 = tid % E4, rl = tid / E4;
            double acc[4] = {0.0, 0.0, 0.0, 0.0};
            const float4* part4 = reinterpret_cast<const float4*>(a.partial);
            for (unsigned p0 = rl; p0 < gridDim.x; p0 += 16 * RL) {
                float4 v[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) {
                    const unsigned p = p0 + u * RL;
                    v[u] = p < gridDim.x ? __ldcg(part4 + (size_t)p * E4 + e4) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int u = 0; u < 16; ++u) { acc[0] += (double)v[u].x; acc[1] += (double)v[u].y; acc[2] += (double)v[u].z; acc[3] += (double)v[u].w; }
            }
            double* sred = reinterpret_cast<double*>(ring);                // RL x 2*C1 doubles = 12 KB (the region is >= 12 KB)
#pragma unroll
            for (int c = 0; c < 4; ++c) sred[(size_t)rl * 2 * C1 + e4 * 4 + c] = acc[c];
            __syncthreads();
            for (int e = tid; e < 2 * C1; e += kF1WThreads) {
                double t = 0.0;
                for (int r = 0; r < RL; ++r) t += sred[(size_t)r * 2 * C1 + e];
                a.stats[e] = (float)t;
            }
            if (tid == 0) g_f1_tickets[a.ticket] = 0u;     // ready for the next launch that draws this ticket
        }
    }
}

// stats[0..C1) = sum, stats[C1..2C1) = sum of squares, over all rows; CTA partials added in index order in fp64
__global__ void f1_stats_reduce_kernel(int nparts, int twoC, const float* __restrict__ partial, float* __restrict__ stats) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= twoC) return;
    double s = 0.0;
    for (int p = 0; p < nparts; ++p) s += (double)partial[(size_t)p * twoC + e];
    stats[e] = (float)s;
}

int launch_dense_raw(long long rows, int K, int N, const float* x, const float* W, float* out, cudaStream_t st);   // below

}  // namespace psa

#include "mlp_internal.cuh"

namespace psa {
int launch_dense_raw(long long rows, int K, int N, const float* x, const float* W, float* out, cudaStream_t st) {
    DenseArgs d;
    d.rows = rows; d.K = K; d.N = N; d.pool_k = 1; d.relu = 0;
    d.x = x; d.W = W; d.scale = nullptr; d.shift = nullptr; d.out = out;
    return launch_dense(d, st);
}
static void f1_grid(int b, int m, int* q_per_cta, dim3* grid) {
    int chunks = (2 * kNumSMs + b - 1) / b;
    int q = (m + chunks - 1) / chunks;
    q = ((q + kF1Warps - 1) / kF1Warps) * kF1Warps;
    if (q < kF1Warps) q = kF1Warps;
    *q_per_cta = q;
    *grid = dim3((m + q - 1) / q, b);
}
}  // namespace psa

using namespace psa;

// streaming kernel: producer layout (NP warps x PPTP points per thread), grid, shared memory, applicability
static bool f1s_plan(int b, int n, int m, int nsample, int* np, int* pptp, int* ctas, size_t* smem) {
    if (n > 4096 || nsample > 128) return false;
    // four search warps (one warpgroup: setmaxnreg is per warpgroup), 32 * 4 * pptp >= n
    *np = kF1NP;
    *pptp = n <= 1024 ? 8 : (n <= 2048 ? 16 : 32);
    *smem = f1s_smem_bytes(n, nsample, *np, *pptp);
    if (*smem > 110 * 1024) return false;
    const long long T = (long long)b * m;
    const long long batches = (T + kF1Batch - 1) / kF1Batch;
    const long long per_sm = 2;                                                   // matches the kernel's __launch_bounds__
    *ctas = (int)(batches < per_sm * kNumSMs ? batches : per_sm * kNumSMs);
    // a whole number of CTAs per cloud when that keeps >= 90 % of the CTA slots busy (the kernel then never crosses a cloud boundary)
    if (b > 0 && *ctas >= b && (*ctas / b) * b * 10 >= *ctas * 9) *ctas = (*ctas / b) * b;
    return true;
}
static bool f1_want_grid(int n, int m) { return bq_grid_fits(n) && n >= 256 && m >= 32; }

extern "C" size_t psa_sa_conv1_prebn_workspace_bytes(int b, int n, int m, int c, int C1, int want_stats) {
    size_t bytes = 0;
    if (c > 0) bytes += ((size_t)b * n * C1 * sizeof(float) + 255) & ~(size_t)255;
    if (want_stats) {
        int q; dim3 g;
        f1_grid(b, m, &q, &g);
        size_t parts = (size_t)g.x * g.y;                                   // round-1 kernel: partials at offset 0
        if (parts < 2 * (size_t)kNumSMs) parts = 2 * (size_t)kNumSMs;      // streaming kernel: up to 2 CTAs per SM, at offset 256
        bytes += parts * 2 * C1 * sizeof(float) + 256;
    }
    return bytes;
}

extern "C" int psa_sa_conv1_prebn(int b, int n, int m, int c, float radius, int nsample, const float* xyz,
                                  const float* new_xyz, const float* points, const float* w1, const float* bias, int C1,
                                  float* pre, int* idx, int* pts_cnt, float* stats, void* workspace,
                                  size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 1 && m >= 0 && c >= 0 && nsample >= 1, "sa_conv1_prebn: bad dims b=%d n=%d m=%d c=%d nsample=%d", b, n, m, c, nsample);
    PSA_REQUIRE(C1 == 64 || C1 == 128, "sa_conv1_prebn: C1=%d must be 64 or 128", C1);
    if (b == 0 || m == 0) return PSA_OK;
    PSA_REQUIRE(xyz && new_xyz && w1 && pre && idx && (points || c == 0), "sa_conv1_prebn: null buffer");
    const size_t need = psa_sa_conv1_prebn_workspace_bytes(b, n, m, c, C1, stats != nullptr);
    PSA_REQUIRE(need == 0 || (workspace != nullptr && workspace_bytes >= need), "sa_conv1_prebn: workspace of %zu bytes required", need);
    cudaStream_t st = as_stream(stream);
    F1Args a;
    a.n = n; a.m = m; a.nsample = nsample; a.C1 = C1;
    bool none = false;
    a.thr = ball_query_threshold(radius, &none);
    a.none = none ? 1 : 0;
    a.radius = radius;
    a.want_grid = f1_want_grid(n, m) ? 1 : 0;
    a.xyz = xyz; a.new_xyz = new_xyz; a.w1 = w1; a.bias = bias; a.pre = pre; a.idx = idx; a.pts_cnt = pts_cnt;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    a.uf = nullptr;
    if (c > 0) {
        int rc = launch_dense_raw((long long)b * n, c, C1, points, w1 + (size_t)3 * C1, reinterpret_cast<float*>(ws), st);
        if (rc != PSA_OK) return rc;
        a.uf = reinterpret_cast<float*>(ws);
        ws += ((size_t)b * n * C1 * sizeof(float) + 255) & ~(size_t)255;
    }
    {   // ---- streaming kernel (persistent CTAs, producer/consumer warps) whenever the cloud fits its shared-memory plan ----
        int ctas = 0, np = 0, pptp = 0;
        size_t ssm = 0;
        if (f1s_plan(b, n, m, nsample, &np, &pptp, &ctas, &ssm)) {
            F1SArgs s;
            s.b = b; s.n = n; s.m = m; s.nsample = nsample; s.C1 = C1; s.thr = a.thr; s.none = a.none;
            s.xyz = xyz; s.new_xyz = new_xyz; s.uf = a.uf; s.w1 = w1; s.bias = bias; s.pre = pre;
            s.idx = idx; s.pts_cnt = pts_cnt; s.partial = nullptr; s.stats = stats; s.ticket = 0;
            if (stats) {
                static std::atomic<unsigned> call_no{0};
                s.ticket = (int)(call_no.fetch_add(1u) % kF1Tickets);
                s.partial = reinterpret_cast<float*>(ws + 256);
            }
#define PSA_F1S_LAUNCH(NV_, U_, PP_)                                                                                          \
    do {                                                                                                                     \
        PSA_CUDA(cudaFuncSetAttribute(sa_conv1_stream_kernel<NV_, U_, PP_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssm)); \
        sa_conv1_stream_kernel<NV_, U_, PP_><<<ctas, kF1WThreads, ssm, st>>>(s);                                             \
    } while (0)
#define PSA_F1S_U(NV_, PP_) do { if (s.uf) PSA_F1S_LAUNCH(NV_, true, PP_); else PSA_F1S_LAUNCH(NV_, false, PP_); } while (0)
#define PSA_F1S_P(NV_)                                                                                                       \
    do {                                                                                                                     \
        if (pptp == 32) PSA_F1S_U(NV_, 32);                                                                                  \
        else if (pptp == 16) PSA_F1S_U(NV_, 16);                                                                             \
        else PSA_F1S_U(NV_, 8);                                                                                              \
    } while (0)
            if (C1 == 64) PSA_F1S_P(2); else PSA_F1S_P(4);
#undef PSA_F1S_P
#undef PSA_F1S_U
#undef PSA_F1S_LAUNCH
            return check_launch("sa_conv1_stream_kernel");
        }
    }
    dim3 grid;
    f1_grid(b, m, &a.q_per_cta, &grid);
    a.partial = stats ? reinterpret_cast<float*>(ws) : nullptr;
    size_t smem = bq_smem_bytes(n, a.want_grid != 0) + (size_t)kF1Warps * ((nsample + 3) & ~3) * sizeof(int) + (stats ? (size_t)kF1Warps * 2 * C1 * sizeof(float) : 0);
    PSA_SUPPORTED(smem <= 200 * 1024, "sa_conv1_prebn: n=%d exceeds the shared-memory resident limit", n);
#define PSA_F1_LAUNCH(NV_, ST_, PPT_)                                                                                        \
    do {                                                                                                                     \
        PSA_CUDA(cudaFuncSetAttribute(sa_conv1_prebn_kernel<NV_, ST_, PPT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        sa_conv1_prebn_kernel<NV_, ST_, PPT_><<<grid, kF1Warps * 32, smem, st>>>(a);                                         \
    } while (0)
#define PSA_F1_DISPATCH(ST_)                                                                                                 \
    do {                                                                                                                     \
        if (n <= 8 * kBqThreads) { if (C1 == 64) PSA_F1_LAUNCH(2, ST_, 8); else PSA_F1_LAUNCH(4, ST_, 8); }                  \
        else { if (C1 == 64) PSA_F1_LAUNCH(2, ST_, 16); else PSA_F1_LAUNCH(4, ST_, 16); }                                    \
    } while (0)
    // shared memory: ball-query arrays, per-warp idx rows, per-warp statistics (16-byte aligned: nsample rows of ints)
    if (stats) {
        PSA_F1_DISPATCH(true);
        f1_stats_reduce_kernel<<<(2 * C1 + 127) / 128, 128, 0, st>>>((int)(grid.x * grid.y), 2 * C1, a.partial, stats);
    } else {
        PSA_F1_DISPATCH(false);
    }
#undef PSA_F1_DISPATCH
#undef PSA_F1_LAUNCH
    return check_launch("sa_conv1_prebn_kernel");
}
