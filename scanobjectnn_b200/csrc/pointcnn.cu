// pointcnn.cu -- PointCNN's X-Conv layer (PointCNN/pointcnn.py:10-52, pointfly.py:122-128, 163-176, 298-347), inference.
//
// What the reference does per layer: a (B,P,N) distance matrix and top_k(K*D) -> every D-th neighbour; gathered (B,P,K,3) local
// coordinates lifted by two dense layers to (B,P,K,C_pts_fts); gathered (B,P,K,C_prev) features; the K x K transformation X from
// a (1,K) conv and two depthwise convs; fts_X = X . F (B,P,K,C_in); a separable (1,K) conv.  Every layer with batch norm has no
// bias and applies ELU before the batch norm: a = elu(x . W) * s + t.
// What happens here:
//   knn_dilated_kernel     one thread per query keeps its K*D nearest in shared memory (sorted, lower index first on ties), in the
//                          canonical fp32 evaluation of oracle/psa_oracle.c:orc_dgcnn_knn, and writes every D-th entry
//   xconv_core_kernel      per tile of queries, everything up to the depthwise stage of the separable conv in shared memory and
//                          registers: only the (B*P, C_in*dm) depthwise output reaches global memory
//   tc_pcnn_dense_kernel   out = elu(x . W [+ bias]) * scale + shift through row strides, on the tensor cores: the shared ring
//                          (ring_gemm.cuh) staging x rows, K padded to 64 by zero operand columns, W padded to a 64- or 128-wide image
//   pcnn_dense_fma_kernel  the same on the fp32 FMA pipe (mode 1, K % 4 != 0, rows < 128, unaligned x)
#include <float.h>

#include "common.cuh"
#include "ring_gemm.cuh"

namespace psa {

using namespace tc;

constexpr int kKnnMaxList = 64;        // k * d entries kept per query
constexpr int kKnnThreads = 128;
constexpr int kXconvMaxK = 16;         // neighbours per query in the core kernel (the fts_X column lives in registers)
constexpr int kXconvThreads = 256;
constexpr int kXconvSmemBudget = 96 * 1024;

__device__ __forceinline__ float elu(float x) { return x > 0.f ? x : expm1f(x); }

// |v|^2 and q . p as fma chains over x, y, z from 0, d = (|q|^2 + (-2 dot)) + |p|^2: the order declared for DGCNN's kNN
// (oracle/psa_oracle.c:orc_dgcnn_knn), here for 3-D points
__device__ __forceinline__ float sq3(float x, float y, float z) { return __fmaf_rn(z, z, __fmaf_rn(y, y, __fmaf_rn(x, x, 0.f))); }
__device__ __forceinline__ float knn_dist3(float qx, float qy, float qz, float sq_q, float px, float py, float pz, float sq_p) {
    const float dot = __fmaf_rn(qz, pz, __fmaf_rn(qy, py, __fmaf_rn(qx, px, 0.f)));
    return __fadd_rn(__fadd_rn(sq_q, __fmul_rn(-2.0f, dot)), sq_p);
}

// ------------------------------------------------------------------------------------------------------------------
// kNN with dilation.  Block (128 queries, cloud); a thread's list is column tid of the (L, 128) shared arrays.  Candidates in
// index order, a candidate enters only if strictly closer than the current last entry, and goes behind entries of equal
// distance: ascending distance, lower index first on ties, as tf.nn.top_k(-D) orders it.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kKnnThreads) knn_dilated_kernel(int n, int m, int k, int d, const float* __restrict__ points,
                                                                  const float* __restrict__ queries, int* __restrict__ idx) {
    extern __shared__ float s_knn[];
    const int L = k * d, tid = threadIdx.x, b = blockIdx.y, qi = blockIdx.x * kKnnThreads + tid;
    float* sd = s_knn;
    int* si = reinterpret_cast<int*>(s_knn + L * kKnnThreads);
    if (qi >= m) return;
    const float* pb = points + (size_t)b * n * 3;
    const float* q = queries + ((size_t)b * m + qi) * 3;
    const float qx = __ldg(q), qy = __ldg(q + 1), qz = __ldg(q + 2), sq_q = sq3(qx, qy, qz);
    int cnt = 0;
    for (int j = 0; j < n; ++j) {
        const float px = __ldg(pb + 3 * j), py = __ldg(pb + 3 * j + 1), pz = __ldg(pb + 3 * j + 2);
        const float dd = knn_dist3(qx, qy, qz, sq_q, px, py, pz, sq3(px, py, pz));
        int pos;
        if (cnt < L) {
            pos = cnt++;
        } else {
            if (!(dd < sd[(L - 1) * kKnnThreads + tid])) continue;
            pos = L - 1;
        }
        while (pos > 0 && sd[(pos - 1) * kKnnThreads + tid] > dd) {
            sd[pos * kKnnThreads + tid] = sd[(pos - 1) * kKnnThreads + tid];
            si[pos * kKnnThreads + tid] = si[(pos - 1) * kKnnThreads + tid];
            --pos;
        }
        sd[pos * kKnnThreads + tid] = dd;
        si[pos * kKnnThreads + tid] = j;
    }
    int* out = idx + ((size_t)b * m + qi) * k;
    for (int s = 0; s < k; ++s) out[s] = si[s * d * kKnnThreads + tid];
}

// ------------------------------------------------------------------------------------------------------------------
// X-Conv core.  Block = QT queries (rows r0 .. r0 + QT of the b*P queries); per query in shared memory: its K neighbour rows,
// the local coordinates (K,3), the first lifting layer (K,Cf), F = [lifted | fts_prev[nn]] (K,C_in), X0 / X2 (K*K) and X1 (K*K).
// Stage loops run over (element, query) with the query fastest, so neighbouring threads read the same weight.
// ------------------------------------------------------------------------------------------------------------------
struct XconvArgs {
    long long rows;               // b * P
    int n, P, K, Cf, Cp, Cin, dm, QT;
    const float* pts;             // (b, n, 3)
    const float* qrs;             // (b, P, 3)
    const int* idx;               // (b*P, K) in [0, n)
    const float* fts;             // (b*n, Cp) or null
    psa_xconv w;
    float* out;                   // (b*P, Cin*dm)
};

__host__ __device__ inline int xconv_query_floats(int K, int Cf, int Cin) { return K + 3 * K + K * Cf + K * Cin + 2 * K * K; }

__global__ void __launch_bounds__(kXconvThreads) xconv_core_kernel(const __grid_constant__ XconvArgs a) {
    extern __shared__ float s_x[];
    const int tid = threadIdx.x, QT = a.QT, K = a.K, Cf = a.Cf, Cin = a.Cin, KK = K * K;
    const long long r0 = (long long)blockIdx.x * QT;
    const int per = xconv_query_floats(K, Cf, Cin);
    // query q's region: nbr (K ints) | local (K,3) | h0 (K,Cf) | F (K,Cin) | XA (K*K) | X1 (K*K)
    auto nbr = [&](int q) { return reinterpret_cast<int*>(s_x + q * per); };
    auto loc = [&](int q) { return s_x + q * per + K; };
    auto h0 = [&](int q) { return s_x + q * per + 4 * K; };
    auto F = [&](int q) { return s_x + q * per + 4 * K + K * Cf; };
    auto XA = [&](int q) { return s_x + q * per + 4 * K + K * Cf + K * Cin; };
    auto X1 = [&](int q) { return s_x + q * per + 4 * K + K * Cf + K * Cin + KK; };
    auto valid = [&](int q) { return r0 + q < a.rows; };

    // ---- neighbours and local coordinates p[nn] - q ----
    for (int e = tid; e < QT * K; e += kXconvThreads) {
        const int q = e % QT, j = e / QT;
        if (!valid(q)) continue;
        const long long r = r0 + q, b = r / a.P;
        const int nb = __ldg(a.idx + r * K + j);
        nbr(q)[j] = nb;
        const float* p = a.pts + ((size_t)b * a.n + nb) * 3;
        const float* c = a.qrs + (size_t)r * 3;
#pragma unroll
        for (int dd = 0; dd < 3; ++dd) loc(q)[j * 3 + dd] = __fsub_rn(__ldg(p + dd), __ldg(c + dd));
    }
    __syncthreads();

    // ---- lifting layer 0 (3 -> Cf), X0 ((K*3) -> K*K), the previous layer's features ----
    for (int e = tid; e < QT * K * Cf; e += kXconvThreads) {
        const int q = e % QT, jc = e / QT, j = jc / Cf, c = jc - j * Cf;
        if (!valid(q)) continue;
        const float* l = loc(q) + j * 3;
        float s = 0.f;
#pragma unroll
        for (int dd = 0; dd < 3; ++dd) s = fmaf(l[dd], __ldg(a.w.w_pts0 + dd * Cf + c), s);
        h0(q)[jc] = fmaf(elu(s), __ldg(a.w.s_pts0 + c), __ldg(a.w.t_pts0 + c));
    }
    for (int e = tid; e < QT * KK; e += kXconvThreads) {
        const int q = e % QT, o = e / QT;
        if (!valid(q)) continue;
        const float* l = loc(q);
        float s = 0.f;
        for (int jd = 0; jd < 3 * K; ++jd) s = fmaf(l[jd], __ldg(a.w.w_x0 + (size_t)jd * KK + o), s);
        XA(q)[o] = fmaf(elu(s), __ldg(a.w.s_x0 + o), __ldg(a.w.t_x0 + o));
    }
    for (int e = tid; e < QT * K * a.Cp; e += kXconvThreads) {
        const int q = e % QT, jc = e / QT, j = jc / a.Cp, c = jc - j * a.Cp;
        if (!valid(q)) continue;
        const long long b = (r0 + q) / a.P;
        F(q)[j * Cin + Cf + c] = __ldg(a.fts + ((size_t)b * a.n + nbr(q)[j]) * a.Cp + c);
    }
    __syncthreads();

    // ---- lifting layer 1 (Cf -> Cf) into F's first Cf columns; X1[b*K + m] = sum_a X0[a*K + b] W1[a][b][m] ----
    for (int e = tid; e < QT * K * Cf; e += kXconvThreads) {
        const int q = e % QT, jc = e / QT, j = jc / Cf, c = jc - j * Cf;
        if (!valid(q)) continue;
        const float* h = h0(q) + j * Cf;
        float s = 0.f;
        for (int i = 0; i < Cf; ++i) s = fmaf(h[i], __ldg(a.w.w_pts1 + i * Cf + c), s);
        F(q)[j * Cin + c] = fmaf(elu(s), __ldg(a.w.s_pts1 + c), __ldg(a.w.t_pts1 + c));
    }
    for (int e = tid; e < QT * KK; e += kXconvThreads) {
        const int q = e % QT, o = e / QT, bb = o / K, mm = o - bb * K;
        if (!valid(q)) continue;
        const float* x0 = XA(q);
        float s = 0.f;
        for (int aa = 0; aa < K; ++aa) s = fmaf(x0[aa * K + bb], __ldg(a.w.w_x1 + (aa * K + bb) * K + mm), s);
        X1(q)[o] = fmaf(elu(s), __ldg(a.w.s_x1 + o), __ldg(a.w.t_x1 + o));
    }
    __syncthreads();

    // ---- X2 (no ELU) over X0's bytes ----
    for (int e = tid; e < QT * KK; e += kXconvThreads) {
        const int q = e % QT, o = e / QT, bb = o / K, mm = o - bb * K;
        if (!valid(q)) continue;
        const float* x1 = X1(q);
        float s = 0.f;
        for (int aa = 0; aa < K; ++aa) s = fmaf(x1[aa * K + bb], __ldg(a.w.w_x2 + (aa * K + bb) * K + mm), s);
        XA(q)[o] = fmaf(s, __ldg(a.w.s_x2 + o), __ldg(a.w.t_x2 + o));
    }
    __syncthreads();

    // ---- fts_X[i][c] = sum_j X2[i][j] F[j][c] (column c in registers), dw[c*dm + m] = sum_i fts_X[i][c] Wdw[i][c][m] ----
    for (int e = tid; e < QT * Cin; e += kXconvThreads) {
        const int q = e % QT, c = e / QT;
        if (!valid(q)) continue;
        const float* x2 = XA(q);
        const float* f = F(q) + c;
        float col[kXconvMaxK];
#pragma unroll
        for (int i = 0; i < kXconvMaxK; ++i) {
            float s = 0.f;
            if (i < K)
                for (int j = 0; j < K; ++j) s = fmaf(x2[i * K + j], f[j * Cin], s);
            col[i] = s;
        }
        float* o = a.out + (size_t)(r0 + q) * Cin * a.dm + (size_t)c * a.dm;
        for (int mm = 0; mm < a.dm; ++mm) {
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < kXconvMaxK; ++i)
                if (i < K) s = fmaf(col[i], __ldg(a.w.w_dw + ((size_t)i * Cin + c) * a.dm + mm), s);
            o[mm] = s;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// tc_pcnn_dense_kernel<NP, NC>: out (rows, N) = elu(x . W + bias) * scale + shift on the ring (ring_gemm.cuh), unit = 128-row tile x
// 64 NC-column tile, all Kp / 64 K blocks.  The producers stage x rows (16 bytes per copy, chunks past K not copied); the consumers
// read the columns past K as zero.
// ------------------------------------------------------------------------------------------------------------------
struct PcnnDenseArgs {
    long long rows, ldx, ldo;
    int K, Kp, N, Np;
    const float* x;            // 16-byte aligned, ldx % 4 == 0 on the tensor path
    const float* bias;         // (N) or null
    const float* scale;        // (N)
    const float* shift;        // (N)
    float* out;
    RingArgs ring;             // W padded to (Kp, Np), format of NP, tile width 64 NC
};

struct PcnnDenseOp {
    const PcnnDenseArgs& a;
    static constexpr bool kClaim = false;
    static constexpr uint32_t kBudget = kRingBudget;
    struct Smem {};
    struct Unit {
        int nb, col0;
        long long r[2];
        bool v[2];
    };

    __device__ int units(int Nt) const { return (int)((a.rows + 127) / 128 * (a.Np / Nt)); }

    template <class Put>
    __device__ void produce(int unit, int Nt, int pw, int lane, Smem&, Put&& put) const {
        const int NTC = a.Np / Nt, KC = a.Kp / 64;
        const long long row0 = (long long)(unit / NTC) * 128;
        const int nt = unit % NTC, r0 = 32 * pw, nr = (int)max(0LL, min(32LL, a.rows - row0 - r0));
        for (int kb = 0; kb < KC; ++kb) put((size_t)nt * KC + kb, [&](uint32_t xs) { stage_rows16(xs, a.x, a.ldx, row0, r0, nr, kb, a.K, lane); });
    }

    __device__ Unit unit(int unit, int Nt, int row, Smem&, int) const {
        const int NTC = a.Np / Nt;
        Unit u;
        u.nb = a.Kp / 64;
        u.col0 = unit % NTC * Nt;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            u.r[i] = (long long)(unit / NTC) * 128 + row + 8 * i;
            u.v[i] = u.r[i] < a.rows;
        }
        return u;
    }

    // rows past `rows` and columns past K read as zero (their staged bytes are stale)
    __device__ void load(const Unit& u, const float* xs, int kb, int t, float2 (&x)[4][2][2]) const {
#pragma unroll
        for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const bool kin = kb * 64 + 16 * s + 8 * h + 2 * t < a.K;     // K % 4 == 0: both columns of the pair or neither
#pragma unroll
                for (int i = 0; i < 2; ++i) x[s][h][i] = u.v[i] && kin ? staged_pair(xs, s, h, i, t) : make_float2(0.f, 0.f);
            }
    }

    // fp16x2 column factor, bias, ELU, the batch-norm affine; only the N real columns are written
    __device__ void epilogue(const Unit& u, const float (&acc)[32], int col0, int t, const float* colscale, Smem&) const {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const int col = col0 + 8 * jj + 2 * t;
            float cs[2] = {1.f, 1.f}, bi[2] = {0.f, 0.f}, sc[2] = {0.f, 0.f}, sh[2] = {0.f, 0.f};
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (col + h < a.N) {
                    if (colscale != nullptr) cs[h] = __ldg(colscale + col + h);
                    if (a.bias != nullptr) bi[h] = __ldg(a.bias + col + h);
                    sc[h] = __ldg(a.scale + col + h);
                    sh[h] = __ldg(a.shift + col + h);
                }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float* o = a.out + (size_t)u.r[i] * a.ldo + col;
                const float y0 = fmaf(elu(fmaf(acc[4 * jj + 2 * i], cs[0], bi[0])), sc[0], sh[0]);
                const float y1 = fmaf(elu(fmaf(acc[4 * jj + 2 * i + 1], cs[1], bi[1])), sc[1], sh[1]);
                if (u.v[i] && col < a.N) o[0] = y0;
                if (u.v[i] && col + 1 < a.N) o[1] = y1;
            }
        }
    }

    __device__ float load_a(long long p, int kk) const { return __ldg(a.x + p * a.ldx + kk); }
    __device__ void store(long long p, int col, float s) const {
        const float bi = a.bias != nullptr ? __ldg(a.bias + col) : 0.f;
        a.out[(size_t)p * a.ldo + col] = fmaf(elu(s + bi), __ldg(a.scale + col), __ldg(a.shift + col));
    }
};

template <int NP, int NC>
__global__ void __launch_bounds__(kRingThreads, 1) tc_pcnn_dense_kernel(const __grid_constant__ PcnnDenseArgs a) {
    ring_gemm<NP, NC>(PcnnDenseOp{a}, a.ring);
}

// the same on the fp32 FMA pipe
__global__ void __launch_bounds__(256) pcnn_dense_fma_kernel(const __grid_constant__ PcnnDenseArgs a, const float* __restrict__ W) {
    fma_gemm(PcnnDenseOp{a}, a.rows, a.K, a.N, W);
}

// ------------------------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------------------------
// the tensor path stages x in 16-byte chunks: K % 4 == 0, ldx % 4 == 0 and x 16-byte aligned (null counts as aligned, so the
// workspace follows from the dims); out, bias, scale and shift are read and written one float at a time
static bool pd_tc_eligible(long long rows, int K, long long ldx, const float* x) {
    return rows >= 128 && K >= 4 && K % 4 == 0 && ldx % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
}
// padded weight image: K to a multiple of 64, N to 64 (N <= 64) or to 64-wide blocks, taken two at a time when their count is even
struct PdPlan {
    int Kp, Np, Nt;
    size_t wp, img2, img3, total;
};
static PdPlan pd_plan(int K, int N, int np) {
    PdPlan p{};
    p.Kp = (K + 63) / 64 * 64;
    const int nb = (N + 63) / 64;
    p.Nt = nb % 2 == 0 ? 128 : 64;
    p.Np = nb * 64;
    size_t off = 256;                                        // word 0: range flag of the fp16x2 launch
    p.wp = off; off += al256((size_t)K * p.Np * sizeof(float));
    if (np == 2) { p.img2 = off; off += tc_image_alloc_bytes(p.Kp, p.Np, 2); }
    p.img3 = off; off += tc_image_alloc_bytes(p.Kp, p.Np, 3);
    p.total = off;
    return p;
}

static const RingKernels kPdRing = {{{(const void*)tc_pcnn_dense_kernel<2, 1>, (const void*)tc_pcnn_dense_kernel<2, 2>},
                                     {(const void*)tc_pcnn_dense_kernel<3, 1>, (const void*)tc_pcnn_dense_kernel<3, 2>}},
                                    "tc_pcnn_dense_kernel", PcnnDenseOp::kBudget};

static int xconv_qt(int K, int Cf, int Cin) {
    const int q = kXconvSmemBudget / (xconv_query_floats(K, Cf, Cin) * (int)sizeof(float));
    return q < 16 ? q : 16;
}

}  // namespace psa

using namespace psa;

extern "C" int psa_knn_dilated(int b, int n, int m, int k, int d, const float* points, const float* queries, int* idx,
                               psa_stream_t stream) {
    PSA_REQUIRE(b >= 0 && n >= 1 && m >= 0 && k >= 1 && d >= 1, "knn_dilated: bad dims b=%d n=%d m=%d k=%d d=%d", b, n, m, k, d);
    PSA_REQUIRE((long long)k * d <= kKnnMaxList, "knn_dilated: k*d = %lld exceeds %d", (long long)k * d, kKnnMaxList);
    PSA_REQUIRE(k * d <= n, "knn_dilated: k*d = %d exceeds the n=%d points (tf.nn.top_k needs that many)", k * d, n);
    PSA_SUPPORTED(b <= 65535, "knn_dilated: b=%d exceeds gridDim.y", b);
    if (b == 0 || m == 0) return PSA_OK;
    PSA_REQUIRE(points && queries && idx, "knn_dilated: null buffer");
    const size_t smem = (size_t)k * d * kKnnThreads * (sizeof(float) + sizeof(int));
    PSA_CUDA(cudaFuncSetAttribute(knn_dilated_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    knn_dilated_kernel<<<dim3((unsigned)((m + kKnnThreads - 1) / kKnnThreads), (unsigned)b), kKnnThreads, smem, as_stream(stream)>>>(
        n, m, k, d, points, queries, idx);
    return check_launch("knn_dilated_kernel");
}

extern "C" int psa_xconv_core(int b, int n, int P, const float* pts, const float* qrs, const int* idx, const float* fts,
                              const psa_xconv* layer, float* out, psa_stream_t stream) {
    PSA_REQUIRE(layer != nullptr, "xconv_core: null layer");
    const psa_xconv& w = *layer;
    PSA_REQUIRE(b >= 0 && n >= 1 && P >= 1, "xconv_core: bad dims b=%d n=%d P=%d", b, n, P);
    PSA_REQUIRE(w.K >= 1 && w.K <= kXconvMaxK && w.K <= n, "xconv_core: K=%d must be in [1, min(%d, n=%d)]", w.K, kXconvMaxK, n);
    PSA_REQUIRE(w.c_pts >= 1 && w.c_prev >= 0 && w.dm >= 1, "xconv_core: bad widths c_pts=%d c_prev=%d dm=%d", w.c_pts, w.c_prev, w.dm);
    PSA_REQUIRE((w.c_prev == 0) == (fts == nullptr), "xconv_core: fts is given exactly when c_prev > 0");
    const int Cin = w.c_pts + w.c_prev;
    PSA_SUPPORTED(xconv_qt(w.K, w.c_pts, Cin) >= 1, "xconv_core: K=%d, C_in=%d exceed the shared-memory budget of one query", w.K, Cin);
    if (b == 0) return PSA_OK;
    PSA_REQUIRE(pts && qrs && idx && out, "xconv_core: null buffer");
    PSA_REQUIRE(w.w_pts0 && w.s_pts0 && w.t_pts0 && w.w_pts1 && w.s_pts1 && w.t_pts1 && w.w_x0 && w.s_x0 && w.t_x0 && w.w_x1 && w.s_x1 &&
                    w.t_x1 && w.w_x2 && w.s_x2 && w.t_x2 && w.w_dw,
                "xconv_core: null weight");
    XconvArgs a;
    a.rows = (long long)b * P; a.n = n; a.P = P; a.K = w.K; a.Cf = w.c_pts; a.Cp = w.c_prev; a.Cin = Cin; a.dm = w.dm;
    a.QT = xconv_qt(w.K, w.c_pts, Cin);
    a.pts = pts; a.qrs = qrs; a.idx = idx; a.fts = fts; a.w = w; a.out = out;
    const size_t smem = (size_t)a.QT * xconv_query_floats(w.K, w.c_pts, Cin) * sizeof(float);
    PSA_CUDA(cudaFuncSetAttribute(xconv_core_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    xconv_core_kernel<<<(unsigned)((a.rows + a.QT - 1) / a.QT), kXconvThreads, smem, as_stream(stream)>>>(a);
    return check_launch("xconv_core_kernel");
}

extern "C" size_t psa_dense_elu_affine_workspace_bytes(long long rows, int K, int N) {
    if (rows < 0 || K < 1 || N < 1) return 0;
    if (mlp_mode() == 1 || !pd_tc_eligible(rows, K, 0, nullptr)) return 0;     // the fp32-FMA kernel needs none
    return pd_plan(K, N, tc_np()).total;
}

extern "C" int psa_dense_elu_affine(long long rows, int K, int N, const float* x, long long ldx, const float* W, const float* bias,
                                    const float* scale, const float* shift, float* out, long long ldo, void* workspace,
                                    size_t workspace_bytes, psa_stream_t stream) {
    PSA_REQUIRE(rows >= 0 && K >= 1 && N >= 1, "dense_elu_affine: bad dims rows=%lld K=%d N=%d", rows, K, N);
    PSA_REQUIRE(ldx >= K && ldo >= N, "dense_elu_affine: row strides ldx=%lld ldo=%lld below K=%d / N=%d", ldx, ldo, K, N);
    PSA_REQUIRE((long long)K * N <= (1LL << 30), "dense_elu_affine: K*N too large");
    if (rows == 0) return PSA_OK;
    PSA_REQUIRE(x && W && scale && shift && out, "dense_elu_affine: null buffer");
    cudaStream_t st = as_stream(stream);
    PcnnDenseArgs a;
    a.rows = rows; a.ldx = ldx; a.ldo = ldo; a.K = K; a.N = N; a.x = x; a.bias = bias; a.scale = scale; a.shift = shift; a.out = out;
    if (mlp_mode() == 1 || !pd_tc_eligible(rows, K, ldx, x)) {
        a.Kp = K; a.Np = N;
        const dim3 grid((unsigned)((rows + 63) / 64), (unsigned)((N + 63) / 64));
        pcnn_dense_fma_kernel<<<grid, 256, 0, st>>>(a, W);
        return check_launch("pcnn_dense_fma_kernel");
    }
    const PdPlan pl = pd_plan(K, N, tc_np());
    PSA_REQUIRE(workspace != nullptr && workspace_bytes >= pl.total,
                "dense_elu_affine: workspace of %zu bytes required (psa_dense_elu_affine_workspace_bytes), got %zu", pl.total, workspace_bytes);
    PSA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "dense_elu_affine: workspace must be 256-byte aligned");
    uint8_t* wsb = reinterpret_cast<uint8_t*>(workspace);
    a.Kp = pl.Kp; a.Np = pl.Np;
    float* wp = reinterpret_cast<float*>(wsb + pl.wp);
    const int rc = pad_cols(K, N, pl.Np, W, wp, st);
    if (rc != PSA_OK) return rc;
    PSA_CUDA(cudaMemsetAsync(wsb, 0, 256, st));
    return ring_run(kPdRing, a, (rows + 127) / 128 * (pl.Np / pl.Nt), RingWeights{K, pl.Kp, pl.Np, pl.Nt, wp, wsb + pl.img2, wsb + pl.img3},
                    reinterpret_cast<unsigned int*>(wsb), nullptr, st);
}
